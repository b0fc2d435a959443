// dfx_search.cu -- the search hot path of one shard on one H100 (sm_90a).
//
// Replaces `self.faiss_index.search(query_batch, top_k)` (reference
// distributed_faiss/index.py:257) for the four builders of index.py:93-100, the factory strings
// of index.py:380-396 and
// `IndexClient._aggregate_results` (client.py:265-310):
//   K1a  gemm_values      coarse quantizer / flat contraction, fp32 FFMA, seq-k canonical order
//   K_sel select_rows     exact k-selection (dfx_select.cuh)
//   K3   pq_prep          per-query PQ table  -2<q_m,P[m][j]>  + exact ||q-c||^2 of probed lists
//   K4   scan_pq          inverted-list scan of PQ codes, per-warp k-selection
//   K4w  scan_pq_wide     64 < M <= 128: table built in shared memory + scan (dfx_scan_pq_wide_dev.cuh)
//   K4n  scan_pq4         4-bit codes: table in registers, lookups by warp shuffle (dfx_scan_pq4_dev.cuh)
//   K_fs pq_fs_lut / scan_pq_fs / fs_dequant   IVF-PQ FastScan: u8 quantized table, integer sums
//                         (dfx_scan_pq_fs_dev.cuh)
//   K2/5 scan_rows        inverted-list scan of fp32 rows / fp16 / 8-bit residual codes
//                         K4n, K_fs and K2/5 share the probe loop and candidate sink of dfx_scan_dev.cuh
//   K_off cand_offsets    k > 1024: slots of each query's candidate row (the list scans then write
//                         every vector's composite, MAT = true, and select_cand picks the k best)
//   K_r  pqr_refine       IVF-PQR: re-ranks the k' = k * k_factor candidates of the IVF-PQ stage on
//                         c + PQ1 + PQ2 (dfx_refine_dev.cuh), then K_sel picks the k best
//   K3f/K4f/K1f pq_flat_lut / pq_flat_topk / pq_flat_values   FLAT_PQ: per-query table, then every
//                         stored code scored per row tile with the tile's top-k fused in (pq_flat_fused:
//                         k <= 100, or nq * k <= 16384), or the values of flat_tiles' column tiles (every
//                         other search, range search)
//                         (dfx_pq_flat_dev.cuh)
//   K_rf rflat_refine     flat refinement (",RFlat"): re-ranks the k' candidates of the base kind's stage
//                         on the stored fp32 rows (dfx_rflat_dev.cuh), then K_sel picks the k best
//   K6   merge            cross-shard merge (float_maxheap_array_t semantics)
// Driver (dfx_search_impl): search_flat, or plan_ivf once per search (every refusal, before any launch)
// and per query chunk (ivf_chunks) K1 -> launch_list_scan -> K_sel / select_cand -> fs_dequant -> refine_candidates.
// Arithmetic orders are the canonical ones of oracle/dfx_oracle.c (bit-exact parity).
#include "dfx_internal.h"
#include "dfx_select.cuh"
#include "dfx_topk.cuh"
#include "dfx_ptx.cuh"
#include <cub/cub.cuh>
#include <cmath>
#include <utility>
#include <vector>

// =====================================================================================
// K1a: values GEMM (fp32 FFMA).  acc = fmaf(q[k], x[k], acc), k ascending.
// =====================================================================================
// The FFMA tile shared by K1a and K7a: the CTA computes rows m0 .. m0 + BM of Q against columns
// n0 .. n0 + BN of X; thread (tx, ty) leaves acc[i][j] = q(m0 + ty TM + i) . x(n0 + tx TN + j).
// X holds fp32 rows, or the fp16 rows of FLAT_SQ16, widened exactly as they are staged.
template <int BM, int BN, int BK, int TM, int TN, class TX>
__device__ __forceinline__ void gemm_tile_ffma(const float* __restrict__ Q, int64_t nq, const TX* __restrict__ X,
                                               int64_t ncols, int d, int64_t m0, int64_t n0, int tx, int ty,
                                               float (&acc)[TM][TN]) {
    constexpr int THREADS = (BM / TM) * (BN / TN);
    __shared__ float sQ[BK][BM + 4];
    __shared__ float sX[BK][BN + 4];
    const int tid = threadIdx.x;
#pragma unroll
    for (int i = 0; i < TM; i++)
#pragma unroll
        for (int j = 0; j < TN; j++) acc[i][j] = 0.f;

    for (int k0 = 0; k0 < d; k0 += BK) {
        for (int e = tid; e < BM * BK; e += THREADS) {
            int m = e / BK, kk = e % BK;
            int64_t gm = m0 + m;
            int gk = k0 + kk;
            sQ[kk][m] = (gm < nq && gk < d) ? Q[gm * d + gk] : 0.f;
        }
        for (int e = tid; e < BN * BK; e += THREADS) {
            int n = e / BK, kk = e % BK;
            int64_t gn = n0 + n;
            int gk = k0 + kk;
            sX[kk][n] = (gn < ncols && gk < d) ? dfx_elem_f32(X[gn * d + gk]) : 0.f;
        }
        __syncthreads();
#pragma unroll
        for (int kk = 0; kk < BK; kk++) {
            float a[TM], b[TN];
#pragma unroll
            for (int i = 0; i < TM; i++) a[i] = sQ[kk][ty * TM + i];
#pragma unroll
            for (int j = 0; j < TN; j++) b[j] = sX[kk][tx * TN + j];
#pragma unroll
            for (int i = 0; i < TM; i++)
#pragma unroll
                for (int j = 0; j < TN; j++) acc[i][j] = __fmaf_rn(a[i], b[j], acc[i][j]);
        }
        __syncthreads();
    }
    // NOTE: zero padding of the k tail adds fmaf(0,0,acc) == acc exactly (acc is never -0 here
    // in a way that matters: acc + (+0) keeps acc), so the canonical order is preserved.
}

template <int BM, int BN, int BK, int TM, int TN, class TX>
__global__ void __launch_bounds__((BM / TM) * (BN / TN))
gemm_values_kernel(const float* __restrict__ Q, int64_t nq, const TX* __restrict__ X,
                   const float* __restrict__ xnorm, int64_t ncols, int d, int metric,
                   float* __restrict__ out, int64_t ld_out) {
    const int tid = threadIdx.x;
    const int tx = tid % (BN / TN), ty = tid / (BN / TN);
    const int64_t m0 = (int64_t)blockIdx.y * BM;
    const int64_t n0 = (int64_t)blockIdx.x * BN;
    float acc[TM][TN];
    gemm_tile_ffma<BM, BN, BK, TM, TN>(Q, nq, X, ncols, d, m0, n0, tx, ty, acc);
#pragma unroll
    for (int i = 0; i < TM; i++) {
        int64_t gm = m0 + ty * TM + i;
        if (gm >= nq) continue;
#pragma unroll
        for (int j = 0; j < TN; j++) {
            int64_t gn = n0 + tx * TN + j;
            if (gn >= ncols) continue;
            out[gm * ld_out + gn] = dfx_rank_value(acc[i][j], metric, xnorm, gn);
        }
    }
}

template <class TX>
static void launch_gemm_values(const float* Q, int64_t nq, const TX* X, const float* xnorm, int64_t ncols, int d,
                               int metric, float* out, int64_t ld_out, cudaStream_t st) {
    if (nq <= 0 || ncols <= 0) return;
    if (nq <= 16) {
        constexpr int BM = 16, BN = 128, BK = 16, TM = 2, TN = 4;
        dim3 grid((unsigned)dfx_ceil_div(ncols, BN), (unsigned)dfx_ceil_div(nq, BM));
        auto kern = gemm_values_kernel<BM, BN, BK, TM, TN, TX>;
        DFX_LAUNCH(kern, grid, (BM / TM) * (BN / TN), 0, st, Q, nq, X, xnorm, ncols, d, metric, out,
                   ld_out);
    } else {
        constexpr int BM = 128, BN = 128, BK = 8, TM = 8, TN = 8;
        dim3 grid((unsigned)dfx_ceil_div(ncols, BN), (unsigned)dfx_ceil_div(nq, BM));
        auto kern = gemm_values_kernel<BM, BN, BK, TM, TN, TX>;
        DFX_LAUNCH(kern, grid, (BM / TM) * (BN / TN), 0, st, Q, nq, X, xnorm, ncols, d, metric, out,
                   ld_out);
    }
}
void dfx_launch_gemm_values(const float* Q, int64_t nq, const float* X, const float* xnorm,
                            int64_t ncols, int d, int metric, float* out, int64_t ld_out,
                            cudaStream_t st) {
    launch_gemm_values(Q, nq, X, xnorm, ncols, d, metric, out, ld_out, st);
}
void dfx_launch_gemm_values(const float* Q, int64_t nq, const __half* X, const float* xnorm,
                            int64_t ncols, int d, int metric, float* out, int64_t ld_out,
                            cudaStream_t st) {
    launch_gemm_values(Q, nq, X, xnorm, ncols, d, metric, out, ld_out, st);
}

// |x|^2 in seq-k order (fp16 rows: of the rows they decode to)
template <class TX>
__global__ void row_norms_kernel(const TX* __restrict__ X, int64_t n, int d,
                                 float* __restrict__ out) {
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const TX* x = X + i * d;
    float acc = 0.f;
    for (int k = 0; k < d; k++) {
        const float v = dfx_elem_f32(x[k]);
        acc = __fmaf_rn(v, v, acc);
    }
    out[i] = acc;
}
void dfx_launch_row_norms(const float* X, int64_t n, int d, float* out, cudaStream_t st) {
    if (n <= 0) return;
    DFX_LAUNCH(row_norms_kernel<float>, (unsigned)dfx_ceil_div(n, 128), 128, 0, st, X, n, d, out);
}
void dfx_launch_row_norms(const __half* X, int64_t n, int d, float* out, cudaStream_t st) {
    if (n <= 0) return;
    DFX_LAUNCH(row_norms_kernel<__half>, (unsigned)dfx_ceil_div(n, 128), 128, 0, st, X, n, d, out);
}

// =====================================================================================
// loaders / writers for the selection kernel
// =====================================================================================
struct ColsLoader {  // a row of a values matrix; sec = col_base + column
    const float* vals;
    int64_t ld;
    uint32_t col_base;
    __device__ __forceinline__ uint64_t operator()(int64_t row, int e) const {
        return dfx_comp(vals[row * ld + e], col_base + (uint32_t)e);
    }
};
struct KeysWriter {  // -> int32 keys (+ optional values, + optional composite copy)
    int32_t* keys;
    float* kvals;
    uint64_t* comp;
    int64_t comp_ld;
    int k;
    __device__ __forceinline__ void operator()(int64_t row, int j, uint64_t c) const {
        if (keys) keys[row * k + j] = (c == DFX_COMP_NONE) ? -1 : (int32_t)(uint32_t)c;
        if (kvals) kvals[row * k + j] = (c == DFX_COMP_NONE) ? FLT_MAX : dfx_key2f((uint32_t)(c >> 32));
        if (comp) comp[row * comp_ld + j] = c;
    }
};
struct CompLoader {  // a row of composites
    const uint64_t* comp;
    int64_t ld;
    __device__ __forceinline__ uint64_t operator()(int64_t row, int e) const {
        return comp[row * ld + e];
    }
};
// the faiss distance of composite c (not DFX_COMP_NONE) of query row `row`: the inner product back
// from its negation (IP), or the L2 value, with |q|^2 added back and clamped at 0 when qnorm is given
// (FLAT L2).  Every result a search or a range search reports goes through here.
__device__ __forceinline__ float dfx_result_distance(uint64_t c, int metric, const float* qnorm, int64_t row) {
    float v = dfx_key2f((uint32_t)(c >> 32));
    if (metric == DFX_METRIC_IP) {
        v = -v;
    } else if (qnorm) {
        v = v + qnorm[row];
        v = v < 0.f ? 0.f : v;
    }
    return v;
}

struct ResultWriter {  // composites -> faiss-style (D, I)
    float* D;
    int64_t* I;
    int k;
    int metric;
    const float* qnorm;          // FLAT L2: add |q|^2 back and clamp at 0
    __device__ __forceinline__ void operator()(int64_t row, int j, uint64_t c) const {
        if (c == DFX_COMP_NONE) {
            D[row * k + j] = (metric == DFX_METRIC_IP) ? -FLT_MAX : FLT_MAX;
            I[row * k + j] = -1;
        } else {
            D[row * k + j] = dfx_result_distance(c, metric, qnorm, row);
            I[row * k + j] = (int64_t)(uint32_t)c;
        }
    }
};

void dfx_launch_select_cols(const float* vals, int64_t nrows, int n, int64_t ld, int k,
                            uint32_t col_base, int32_t* keys, float* kvals, uint64_t* comp_out,
                            int64_t comp_ld, cudaStream_t st) {
    ColsLoader ldr{vals, ld, col_base};
    KeysWriter wr{keys, kvals, comp_out, comp_ld, k};
    dfx_launch_select<256>(ldr, wr, nrows, n, k, st);
}

void dfx_launch_select_comp(const uint64_t* comp, int64_t nrows, int n, int64_t ld, int k, int32_t* keys,
                            cudaStream_t st) {
    CompLoader ldr{comp, ld};
    KeysWriter wr{keys, nullptr, nullptr, 0, k};
    dfx_launch_select<256>(ldr, wr, nrows, n, k, st);
}

#include "dfx_pq_prep_dev.cuh"
#include "dfx_scan_dev.cuh"
#include "dfx_scan_pq_wide_dev.cuh"
#include "dfx_scan_pq4_dev.cuh"
#include "dfx_scan_pq_fs_dev.cuh"
#include "dfx_refine_dev.cuh"
#include "dfx_rflat_dev.cuh"
#include "dfx_pq_flat_dev.cuh"

// =====================================================================================
// K4: scan_pq.  one CTA = (query, group of G consecutive probes).  lane-per-vector:
//   v = dis0 + (t + S),  S = halving-tree sum of lut[m][code_m] (oracle pq_sum)
// =====================================================================================
// The probe loop, the walk and the candidate sink are the list-scan skeleton (dfx_scan_dev.cuh).
// <0, false>: asking for 6 resident blocks keeps it at 80 registers (92 by default); the rest keep 0.
template <int MT, bool MAT = false>
__global__ void __launch_bounds__(128, (MT == 0 && !MAT) ? 6 : 0)
scan_pq_kernel(const float* __restrict__ lut, const float* __restrict__ dis0,
               const int32_t* __restrict__ keys, int nprobe, int G, int ngroups,
               const int64_t* __restrict__ list_off, const uint8_t* __restrict__ codes,
               const float* __restrict__ tvals, const int32_t* __restrict__ ids, int Mrt, int ksub,
               int k, int cap, uint64_t* __restrict__ part, const int64_t* __restrict__ coff) {
    DFX_DYN_SMEM(unsigned char, smem_raw, 16);
    const int M = (MT > 0) ? MT : Mrt;
    float* s_lut = reinterpret_cast<float*>(smem_raw);
    const ScanProbes pr(keys, dis0, list_off, nprobe, G, ngroups);

    {
        const float4* src = reinterpret_cast<const float4*>(lut + pr.q * (int64_t)M * ksub);
        float4* dst = reinterpret_cast<float4*>(s_lut);
        for (int i = threadIdx.x; i < (M * ksub) / 4; i += 128) dst[i] = src[i];
    }
    ScanSink<MAT, 128> sink(reinterpret_cast<uint64_t*>(smem_raw + (size_t)M * ksub * 4), cap, k, part, coff);
    __syncthreads();

    dfx_scan_lanes<true>(pr, sink, [&](int64_t i, bool valid, int64_t base, float d0) {
        // MT = 0: tail lanes compute on the warp's first row, so that the sink's admission is the only test
        // of `valid` (0.6 % faster on an H100); the 16-byte loads of MT > 0 run 8-12 % faster under if (valid)
        if (MT == 0) {
            i = valid ? i : base;
            valid = true;
        }
        float v = 0.f;
        uint32_t my_id = DFX_SEC_NONE;  // loaded with the code: never a dependent load on admission
        if (valid) {
            my_id = (uint32_t)__ldg(ids + i);
            // table values of this vector, then the canonical halving tree (oracle pq_sum)
            constexpr int P = (MT > 0) ? MT : 64;  // MT is a power of two when > 0
            float val[P];
            if (MT > 0 && (MT % 16) == 0) {
                const uint4* cp = reinterpret_cast<const uint4*>(codes + i * (int64_t)M);
#pragma unroll
                for (int w4 = 0; w4 < MT / 16; w4++) {
                    uint4 c = __ldg(cp + w4);
                    uint32_t wv[4] = {c.x, c.y, c.z, c.w};
#pragma unroll
                    for (int w = 0; w < 4; w++) {
                        const int m = w4 * 16 + w * 4;
                        val[m + 0] = s_lut[(m + 0) * ksub + (wv[w] & 255u)];
                        val[m + 1] = s_lut[(m + 1) * ksub + ((wv[w] >> 8) & 255u)];
                        val[m + 2] = s_lut[(m + 2) * ksub + ((wv[w] >> 16) & 255u)];
                        val[m + 3] = s_lut[(m + 3) * ksub + (wv[w] >> 24)];
                    }
                }
            } else {
                const uint32_t* cp = reinterpret_cast<const uint32_t*>(codes + i * (int64_t)M);
#pragma unroll
                for (int w = 0; w < P / 4; w++) {
                    const int m = w * 4;
                    if (m < M) {
                        uint32_t c = __ldg(cp + w);
                        val[m + 0] = s_lut[(m + 0) * ksub + (c & 255u)];
                        val[m + 1] = s_lut[(m + 1) * ksub + ((c >> 8) & 255u)];
                        val[m + 2] = s_lut[(m + 2) * ksub + ((c >> 16) & 255u)];
                        val[m + 3] = s_lut[(m + 3) * ksub + (c >> 24)];
                    } else {
                        val[m + 0] = val[m + 1] = val[m + 2] = val[m + 3] = 0.f;
                    }
                }
            }
            dfx_halving_tree<P / 2>(val);
            v = d0 + (__ldg(tvals + i) + val[0]);
        }
        return ScanCand{v, my_id};
    });
    sink.finish(pr);
}

// =====================================================================================
// K2 / K5: scan_rows.  warp-per-vector, warp-dot canonical order.
//   MODE 0: fp32 rows, value = -<q,x>      (IVF-Flat, IP)
//   MODE 1: fp32 rows, value = ||q-x||^2   (IVF-Flat, L2)
//   MODE 2: fp16 residual codes, value = ||(q-c) - half2float(code)||^2   (IVF-SQ fp16)
//   MODE 3: 8-bit residual codes, value = ||(q-c) - dfx_sq8_decode(code)||^2   (IVF-SQ8)
// =====================================================================================
// U = vectors in flight per warp: 4 (default), 8 = EXPERIMENTAL (dfx_set_param "rows_inflight"):
// the kernel is bound by memory-level parallelism, not by instructions -- on a B200, C2 (512 B per
// vector) reached 0.46 of the HBM peak and C4 (1536 B per vector) 0.68 with the same code.
//
// MODE 3 decodes faiss's QT_8bit component (AVX2 form, DESIGN.md section 2):
//   t = fmaf(code, 1/255, 0.5/255),  x = fmaf(t, vdiff, vmin).
// (float)code is built as 0x4B0000cc - 2^23 (one PRMT + one FADD, exact) instead of an I2F, which
// issues at an eighth of the FFMA rate on sm_90.  `sel` picks code byte j: 0x7540 + j.
__device__ __forceinline__ float dfx_sq8_component(uint32_t w, uint32_t sel, float vmin, float vdiff) {
    const float c = __uint_as_float(__byte_perm(w, 0x4B000000u, sel)) - 8388608.f;
    return __fmaf_rn(__fmaf_rn(c, DFX_SQ8_SCALE, DFX_SQ8_BIAS), vdiff, vmin);
}

template <int MODE, int U = 4, bool MAT = false>
__global__ void __launch_bounds__(128)
scan_rows_kernel(const float* __restrict__ Q, int d, const float* __restrict__ cent,
                 const int32_t* __restrict__ keys, int nprobe, int G, int ngroups,
                 const int64_t* __restrict__ list_off, const void* __restrict__ rows,
                 const int32_t* __restrict__ ids, int k, int cap, uint64_t* __restrict__ part,
                 const float* __restrict__ sq_trained, const int64_t* __restrict__ coff) {
    DFX_DYN_SMEM(unsigned char, smem_raw, 16);
    float* s_q = reinterpret_cast<float*>(smem_raw);   // query (MODE 2 / 3: residual q - c)
    float* s_q0 = s_q + d;                              // MODE 2 / 3: the raw query
    float* s_vmin = s_q + 2 * d;                        // MODE 3: vmin, then vdiff
    float* s_vdiff = s_q + 3 * d;
    const int dpad = (MODE == 3) ? 4 * d : (MODE == 2) ? 2 * d : d;
    const ScanProbes pr(keys, nullptr, list_off, nprobe, G, ngroups);
    const int64_t q = pr.q;
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;

    for (int i = tid; i < d; i += 128) {
        float qv = Q[q * d + i];
        s_q[i] = qv;
        if (MODE >= 2) s_q0[i] = qv;
        if (MODE == 3) {
            s_vmin[i] = sq_trained[i];
            s_vdiff[i] = sq_trained[d + i];
        }
    }
    ScanSink<MAT, 128> sink(reinterpret_cast<uint64_t*>(smem_raw + (((size_t)dpad * 4 + 15) / 16) * 16), cap, k,
                            part, coff);
    __syncthreads();

    const auto residual = [&](int l) {
        if (MODE >= 2) {
            __syncthreads();
            for (int i = tid; i < d; i += 128) s_q[i] = s_q0[i] - cent[(size_t)l * d + i];
            __syncthreads();
        }
    };
    pr.for_each_list<false>(sink, residual, [&](int64_t beg, int64_t end, float) {
        for (int64_t base = beg + warp * U; base < end; base += 4 * U) {
            float acc[U];
            uint32_t vid[U];
#pragma unroll
            for (int u = 0; u < U; u++) {
                acc[u] = 0.f;
                vid[u] = (base + u < end) ? (uint32_t)__ldg(ids + base + u) : DFX_SEC_NONE;
            }
            for (int kb = 4 * lane; kb < d; kb += 128) {
                const float4 qv = *reinterpret_cast<const float4*>(s_q + kb);
                float4 xv[U];
                if (MODE == 3) {
                    // 4 code bytes per lane and vector: a warp reads 128 contiguous bytes per vector
                    uint32_t cw[U];
#pragma unroll
                    for (int u = 0; u < U; u++) {
                        const int64_t i = base + u;
                        cw[u] = (i < end) ? __ldg(reinterpret_cast<const uint32_t*>(
                                                reinterpret_cast<const uint8_t*>(rows) + i * (int64_t)d + kb))
                                          : 0u;
                    }
                    const float4 vmn = *reinterpret_cast<const float4*>(s_vmin + kb);
                    const float4 vdf = *reinterpret_cast<const float4*>(s_vdiff + kb);
#pragma unroll
                    for (int u = 0; u < U; u++) {
                        xv[u] = make_float4(dfx_sq8_component(cw[u], 0x7540u, vmn.x, vdf.x),
                                            dfx_sq8_component(cw[u], 0x7541u, vmn.y, vdf.y),
                                            dfx_sq8_component(cw[u], 0x7542u, vmn.z, vdf.z),
                                            dfx_sq8_component(cw[u], 0x7543u, vmn.w, vdf.w));
                    }
                } else {
#pragma unroll
                for (int u = 0; u < U; u++) {
                    const int64_t i = base + u;
                    if (i < end) {
                        if (MODE == 2) {
                            const uint2 h = __ldg(reinterpret_cast<const uint2*>(
                                reinterpret_cast<const __half*>(rows) + i * (int64_t)d + kb));
                            const __half2 h01 = *reinterpret_cast<const __half2*>(&h.x);
                            const __half2 h23 = *reinterpret_cast<const __half2*>(&h.y);
                            const float2 f01 = __half22float2(h01), f23 = __half22float2(h23);
                            xv[u] = make_float4(f01.x, f01.y, f23.x, f23.y);
                        } else {
                            xv[u] = __ldg(reinterpret_cast<const float4*>(
                                reinterpret_cast<const float*>(rows) + i * (int64_t)d + kb));
                        }
                    } else {
                        xv[u] = make_float4(0.f, 0.f, 0.f, 0.f);
                    }
                }
                }
#pragma unroll
                for (int u = 0; u < U; u++) {
                    if (MODE == 0) {
                        acc[u] = __fmaf_rn(qv.x, xv[u].x, acc[u]);
                        acc[u] = __fmaf_rn(qv.y, xv[u].y, acc[u]);
                        acc[u] = __fmaf_rn(qv.z, xv[u].z, acc[u]);
                        acc[u] = __fmaf_rn(qv.w, xv[u].w, acc[u]);
                    } else {
                        float df;
                        df = qv.x - xv[u].x; acc[u] = __fmaf_rn(df, df, acc[u]);
                        df = qv.y - xv[u].y; acc[u] = __fmaf_rn(df, df, acc[u]);
                        df = qv.z - xv[u].z; acc[u] = __fmaf_rn(df, df, acc[u]);
                        df = qv.w - xv[u].w; acc[u] = __fmaf_rn(df, df, acc[u]);
                    }
                }
            }
#pragma unroll
            for (int u = 0; u < U; u++) {
                const int64_t i = base + u;
                float v = dfx_warp_butterfly(acc[u]);
                if (MODE == 0) v = -v;
                sink.push_uniform(i < end, u, i, v, vid[u]);
            }
        }
    });
    sink.finish(pr);
}

// =====================================================================================
// K6: cross-shard merge (client.py:265-310 / float_maxheap_array_t)
// =====================================================================================
struct MergeLoader {
    const float* D;
    int64_t nq;
    int k;
    int negate;
    __device__ __forceinline__ uint64_t operator()(int64_t row, int e) const {
        int s = e / k, j = e - s * k;
        float v = D[((int64_t)s * nq + row) * k + j];
        if (negate) v = -v;
        if (!(v < FLT_MAX)) return DFX_COMP_NONE;  // heapify(): admitted only if FLT_MAX > v
        return dfx_comp(v, (uint32_t)e);
    }
};
struct MergeWriter {
    const int64_t* I;
    int64_t nq;
    int k;
    float* outD;
    int64_t* outI;
    __device__ __forceinline__ void operator()(int64_t row, int j, uint64_t c) const {
        if (c == DFX_COMP_NONE) {
            outD[row * k + j] = FLT_MAX;
            outI[row * k + j] = -1;
        } else {
            uint32_t e = (uint32_t)c;
            int s = e / k, jj = e - s * k;
            outD[row * k + j] = dfx_key2f((uint32_t)(c >> 32));
            outI[row * k + j] = I[((int64_t)s * nq + row) * k + jj];
        }
    }
};

void dfx_merge_impl(int64_t S, int64_t nq, int64_t k, const float* d_D, const int64_t* d_I,
                    int negate, float* d_outD, int64_t* d_outI, cudaStream_t st) {
    DFX_REQUIRE(S >= 1 && k >= 1 && S * k < (1ll << 31), "merge: bad S/k");
    if (nq <= 0) return;
    MergeLoader ldr{d_D, nq, (int)k, negate};
    MergeWriter wr{d_I, nq, (int)k, d_outD, d_outI};
    dfx_launch_select<128>(ldr, wr, nq, (int)(S * k), (int)k, st);
}

__global__ void map_ids_kernel(int64_t n, const int64_t* __restrict__ ids,
                               const int64_t* __restrict__ table, int64_t* __restrict__ out) {
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) {
        int64_t v = ids[i];
        out[i] = v < 0 ? -1 : table[v];
    }
}
void dfx_map_ids_impl(int64_t n, const int64_t* d_ids, const int64_t* d_table, int64_t* d_out,
                      cudaStream_t st) {
    if (n <= 0) return;
    DFX_LAUNCH(map_ids_kernel, (unsigned)dfx_ceil_div(n, 256), 256, 0, st, n, d_ids, d_table, d_out);
}

// ---- packed exchange form: what ONE all-gather over the ranks delivers.  Rank r's block starts at
// base + r * rank_stride and holds D f32[S_loc][nq][k] at offset 0 and I i64[S_loc][nq][k] at
// off_I.  Shard s = r * S_loc + j (rank-major), same total order as dfx_merge_impl.
struct MergePackedLoader {
    const unsigned char* base;
    int64_t rank_stride, nq;
    int k, s_loc, negate;
    __device__ __forceinline__ uint64_t operator()(int64_t row, int e) const {
        int s = e / k, j = e - s * k;
        int r = s / s_loc, sl = s - r * s_loc;
        const float* D = reinterpret_cast<const float*>(base + (int64_t)r * rank_stride);
        float v = D[((int64_t)sl * nq + row) * k + j];
        if (negate) v = -v;
        if (!(v < FLT_MAX)) return DFX_COMP_NONE;
        return dfx_comp(v, (uint32_t)e);
    }
};
struct MergePackedWriter {
    const unsigned char* base;
    int64_t rank_stride, off_I, nq;
    int k, s_loc;
    float* outD;
    int64_t* outI;
    __device__ __forceinline__ void operator()(int64_t row, int j, uint64_t c) const {
        if (c == DFX_COMP_NONE) {
            outD[row * k + j] = FLT_MAX;
            outI[row * k + j] = -1;
        } else {
            uint32_t e = (uint32_t)c;
            int s = e / k, jj = e - s * k;
            int r = s / s_loc, sl = s - r * s_loc;
            const int64_t* I = reinterpret_cast<const int64_t*>(base + (int64_t)r * rank_stride + off_I);
            outD[row * k + j] = dfx_key2f((uint32_t)(c >> 32));
            outI[row * k + j] = I[((int64_t)sl * nq + row) * k + jj];
        }
    }
};
void dfx_merge_packed_impl(int64_t R, int64_t S_loc, int64_t nq, int64_t k, const void* d_packed,
                           int64_t rank_stride, int64_t off_I, int negate, float* d_outD,
                           int64_t* d_outI, cudaStream_t st) {
    DFX_REQUIRE(R >= 1 && S_loc >= 1 && k >= 1 && R * S_loc * k < (1ll << 31), "merge: bad R/S/k");
    DFX_REQUIRE(rank_stride % 8 == 0 && off_I % 8 == 0 && off_I >= S_loc * nq * k * 4,
                "merge: the packed blocks must be 8-byte aligned and I must follow D");
    if (nq <= 0) return;
    const unsigned char* b = reinterpret_cast<const unsigned char*>(d_packed);
    MergePackedLoader ldr{b, rank_stride, nq, (int)k, (int)S_loc, negate};
    MergePackedWriter wr{b, rank_stride, off_I, nq, (int)k, (int)S_loc, d_outD, d_outI};
    dfx_launch_select<128>(ldr, wr, nq, (int)(R * S_loc * k), (int)k, st);
}

// shard-local ids -> exchange ids: (shard tag << 40) | local id, -1 stays -1.  With a metadata
// column (int32 code per local id; -2 = the entry has no such metadata position) the entries the
// reference's post-filter would drop (client.py:235-243: meta[filter_pos] == filter_value, or no
// metadata / too short) get bit 62 set; the flag rides through all-gather + merge untouched.
__global__ void encode_ids_kernel(int64_t n, const int64_t* __restrict__ ids, int64_t tag,
                                  const int32_t* __restrict__ col, int32_t drop_code,
                                  int64_t* __restrict__ out) {
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    int64_t v = ids[i];
    if (v < 0) {
        out[i] = -1;
        return;
    }
    int64_t e = (tag << 40) | v;
    if (col) {
        int32_t c = col[v];
        if (c == drop_code || c == -2) e |= (1ll << 62);
    }
    out[i] = e;
}
void dfx_encode_ids_impl(int64_t n, const int64_t* d_ids, int64_t tag, const int32_t* d_col,
                         int32_t drop_code, int64_t* d_out, cudaStream_t st) {
    DFX_REQUIRE(tag >= 0 && tag < (1ll << 20), "encode_ids: shard tag out of range");
    if (n <= 0) return;
    DFX_LAUNCH(encode_ids_kernel, (unsigned)dfx_ceil_div(n, 256), 256, 0, st, n, d_ids, tag, d_col, drop_code, d_out);
}

// post-filter of search_with_filter on device (client.py:229-250): per query walk the kin merged
// slots in rank order, keep the entries that exist (I >= 0) and do not carry the drop flag, stop
// at kout.  One warp per query; ballot + prefix popcount keeps the order.
__global__ void filter_compact_kernel(int64_t nq, int kin, int kout, const float* __restrict__ D,
                                      const int64_t* __restrict__ I, float* __restrict__ outD,
                                      int64_t* __restrict__ outI, int32_t* __restrict__ outCount) {
    const int64_t q = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (q >= nq) return;
    int kept = 0;
    for (int j0 = 0; j0 < kin && kept < kout; j0 += 32) {
        int j = j0 + lane;
        int64_t id = (j < kin) ? I[q * kin + j] : -1;
        bool keep = id >= 0 && !(id & (1ll << 62));
        unsigned m = __ballot_sync(0xffffffffu, keep);
        int pos = kept + __popc(m & ((1u << lane) - 1u));
        if (keep && pos < kout) {
            outD[q * kout + pos] = D[q * kin + j];
            outI[q * kout + pos] = id;
        }
        kept += __popc(m);
    }
    if (kept > kout) kept = kout;
    for (int j = kept + lane; j < kout; j += 32) {
        outD[q * kout + j] = FLT_MAX;
        outI[q * kout + j] = -1;
    }
    if (lane == 0) outCount[q] = kept;
}
void dfx_filter_compact_impl(int64_t nq, int64_t kin, int64_t kout, const float* d_D, const int64_t* d_I,
                             float* d_outD, int64_t* d_outI, int32_t* d_count, cudaStream_t st) {
    DFX_REQUIRE(kin >= 1 && kout >= 1 && kin < (1 << 20), "filter: bad k");
    if (nq <= 0) return;
    DFX_LAUNCH(filter_compact_kernel, (unsigned)dfx_ceil_div(nq, 4), 128, 0, st, nq, (int)kin, (int)kout, d_D, d_I,
               d_outD, d_outI, d_count);
}

// ndis of the last search = sum over (q,p) of len(list keys[q][p])
__global__ void ndis_kernel(const int32_t* __restrict__ keys, int64_t n,
                            const int64_t* __restrict__ list_off, unsigned long long* out) {
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    unsigned long long v = 0;
    if (i < n) {
        int l = keys[i];
        if (l >= 0) v = (unsigned long long)(list_off[l + 1] - list_off[l]);
    }
    for (int off = 16; off >= 1; off >>= 1) v += __shfl_xor_sync(0xffffffffu, v, off);
    if ((threadIdx.x & 31) == 0 && v) atomicAdd(out, v);
}
void dfx_stats_impl(dfx_index* idx, int64_t* ndis, cudaStream_t st) {
    *ndis = 0;
    if (!idx->is_ivf() || !idx->last_keys_valid) return;
    int64_t n = idx->last_nq * idx->last_nprobe;
    if (n <= 0) return;
    idx->w_misc.reserve(8);
    DFX_CUDA(cudaMemsetAsync(idx->w_misc.p, 0, 8, st));
    DFX_LAUNCH(ndis_kernel, (unsigned)dfx_ceil_div(n, 256), 256, 0, st, idx->w_keys.as<int32_t>(), n,
               idx->list_off.as<int64_t>(), idx->w_misc.as<unsigned long long>());
    unsigned long long h = 0;
    DFX_CUDA(cudaMemcpyAsync(&h, idx->w_misc.p, 8, cudaMemcpyDeviceToHost, st));
    DFX_CUDA(cudaStreamSynchronize(st));
    *ndis = (int64_t)h;
}

// =====================================================================================
// k > 1024.  The per-warp queues of the list scans would need 4 x 2 KP x 8 B of shared memory per
// CTA (256 KiB at k = 4096), so the scans write the composite of every probed vector instead
// (MAT = true) and one k-selection per query picks the result.  Row q of a query chunk holds its
// probed lists end to end from slot q * ld; ld, the nprobe longest lists of the index together,
// bounds every row and is known on the host, so nothing is read back from the device.
// =====================================================================================
// coff[q][p] = q * ld + (vectors in the lists of probes < p), coff[q][nprobe] = q * ld + n_q; a
// missing probe (key < 0) holds none.  One warp per query; lane j sums a contiguous run of probes.
__global__ void __launch_bounds__(128)
cand_offsets_kernel(const int32_t* __restrict__ keys, int64_t nq, int nprobe, const int64_t* __restrict__ list_off,
                    int64_t ld, int64_t* __restrict__ coff) {
    const int64_t q = (int64_t)blockIdx.x * 4 + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (q >= nq) return;  // warp-uniform
    const int per = (nprobe + 31) / 32;
    const int p0 = min(nprobe, lane * per), p1 = min(nprobe, p0 + per);
    const int32_t* kq = keys + q * nprobe;
    auto len = [&](int p) -> long long {
        const int l = kq[p];
        return l < 0 ? 0ll : (long long)(list_off[l + 1] - list_off[l]);
    };
    long long s = 0;
    for (int p = p0; p < p1; p++) s += len(p);
    long long incl = s;  // inclusive prefix over the lanes
    for (int off = 1; off < 32; off <<= 1) {
        const long long o = __shfl_sync(0xffffffffu, incl, lane >= off ? lane - off : 0);
        if (lane >= off) incl += o;
    }
    int64_t* out = coff + q * (nprobe + 1);
    long long c = q * ld + (incl - s);
    for (int p = p0; p < p1; p++) {
        out[p] = c;
        c += len(p);
    }
    if (lane == 31) out[nprobe] = q * ld + incl;
}

struct SlotLoader {  // one candidate row
    const uint64_t* c;
    __device__ __forceinline__ uint64_t operator()(int64_t, int e) const { return c[e]; }
};
// one CTA per query: the k best of its n_q candidates, each row with its own length
template <int THREADS>
__global__ void __launch_bounds__(THREADS)
select_cand_kernel(const uint64_t* __restrict__ cand, const int64_t* __restrict__ coff, int nprobe, ResultWriter wr,
                   int k, int P, int sort_cap) {
    DFX_DYN_SMEM(unsigned char, smem_raw, 16);
    const int64_t q = blockIdx.x;
    const int64_t b = coff[q * (nprobe + 1)], n = coff[q * (nprobe + 1) + nprobe] - b;
    dfx_select_row<THREADS>(SlotLoader{cand + b}, wr, q, (int)n, k, P, sort_cap, reinterpret_cast<uint64_t*>(smem_raw));
}

// =====================================================================================
// IVF-PQR and the flat refinement: re-rank the k1 = k' candidates of each query of a chunk (cand
// [qc][k1], the ids the first stage selected) and select the k best into (D, I) -- the order and
// the padding are those of every other kind.  Bracketed by the refine profiling range
// (dfx_get_param "refine_ms").
// =====================================================================================
static void refine_candidates(dfx_index* idx, const float* xq, int64_t qc, int k1, int k, const int64_t* cand,
                              float* D, int64_t* I, cudaStream_t st) {
    if (idx->prof_on) idx->prof_refine.begin(st);
    const int64_t nc = qc * k1;
    uint64_t* comp = idx->w_rcomp.as<uint64_t>();
    if (idx->rflat()) {
        // exact distances on the stored fp32 rows; rows of up to 1 KB: two candidates per warp in flight
        const int d = idx->cfg.d;
        const int U = (size_t)d * 4 <= 1024 ? 2 : 1;
        const int cpq = (k1 + RFLAT_WARPS * U - 1) / (RFLAT_WARPS * U);
        auto kern = U == 2 ? rflat_refine_kernel<2> : rflat_refine_kernel<1>;
        DFX_LAUNCH(kern, (unsigned)(qc * cpq), 32 * RFLAT_WARPS, (size_t)d * 4, st, xq, d, k1, cpq, cand,
                   idx->refine_vecs.as<float>(), comp);
    } else {
        const int il = idx->il ? 1 : 0;
        DFX_LAUNCH(pqr_refine_kernel, (unsigned)dfx_ceil_div(nc, PQR_WARPS), 32 * PQR_WARPS, 0, st, xq, idx->cfg.d, nc,
                   k1, cand, idx->inv.as<int32_t>(), il ? idx->blk_off.as<int64_t>() : idx->list_off.as<int64_t>(),
                   idx->cfg.nlist, il, il ? idx->il_codes.as<uint8_t>() : idx->payload.as<uint8_t>(), idx->M,
                   idx->dsub, idx->codebooks.as<float>(), idx->refine_codes.as<uint8_t>(), idx->M2, idx->dsub2,
                   idx->refine_cb.as<float>(), idx->centroids.as<float>(), comp);
    }
    CompLoader ldr{comp, k1};
    ResultWriter wr{D, I, k, DFX_METRIC_L2, nullptr};
    dfx_launch_select<128>(ldr, wr, qc, k1, k, st);
    if (idx->prof_on) idx->prof_refine.end(st);
}

// =====================================================================================
// the per-shard search driver
// =====================================================================================
static int choose_group(int64_t nq, int nprobe) {
    // keep >= ~8 CTAs per SM in flight; at large batch let one CTA walk several lists so the
    // query's table is staged into shared memory once.
    const int64_t target = (int64_t)dfx_num_sms() * 8;
    int64_t G = (nq * (int64_t)nprobe) / target;
    if (G < 1) G = 1;
    if (G > nprobe) G = nprobe;
    if (G > 16) G = 16;
    return (int)G;
}

// FLAT / FLAT_SQ16 L2: |q|^2 of every query into buf, added back to the distances the search reports; nullptr for
// inner product
static const float* query_norms(dfx_index* idx, int64_t nq, const float* d_x, DevBuf& buf, cudaStream_t st) {
    if (idx->cfg.metric != DFX_METRIC_L2 || !idx->flat_rows()) return nullptr;  // FLAT_PQ: the table holds all of it
    buf.reserve((size_t)nq * 4);
    dfx_launch_row_norms(d_x, nq, idx->cfg.d, buf.as<float>(), st);
    return buf.as<float>();
}

static constexpr int64_t kFlatTile = 32768;

// ---- FLAT_PQ (dfx_pq_flat_dev.cuh)
// f(MT, WIDE) for the instantiation that serves M: M = 8, 16, 32, 64, 96, 128 have their own code width,
// any other M % 4 == 0 takes the generic shape of its half (M <= 64: P = 64; 64 < M <= 128: P = 128)
template <class F>
static void pq_flat_dispatch(int M, F&& f) {
    if (M > 64) {
        if (!dispatch_int(IntList<128, 96>{}, M, [&](auto MT) { f(MT, std::true_type{}); }))
            f(std::integral_constant<int, 0>{}, std::true_type{});
    } else if (!dispatch_int(IntList<8, 16, 32, 64>{}, M, [&](auto MT) { f(MT, std::false_type{}); })) {
        f(std::integral_constant<int, 0>{}, std::false_type{});
    }
}

// rows per CTA of the FLAT_PQ scoring kernels over n rows for qc queries: kFlatTile, halved (down to
// 2048) while the grid would hold fewer than 4 CTAs per SM, so that small batches still fill the device
static int64_t pq_flat_span(int64_t qc, int64_t n) {
    int64_t r = kFlatTile;
    while (r > 2048 && qc * dfx_ceil_div(n, r) < 4ll * dfx_num_sms()) r >>= 1;
    return r;
}

// K3f: the [M][256] table of each of the qc queries xq into w_lut
static void pq_flat_tables(dfx_index* idx, const float* xq, int64_t qc, cudaStream_t st) {
    idx->w_lut.reserve((size_t)qc * idx->M * PQF_KSUB * 4);
    DFX_LAUNCH(pq_flat_lut_kernel, (unsigned)qc, 256, 0, st, xq, idx->cfg.d, idx->M, idx->dsub,
               idx->codebooks.as<float>(), idx->cfg.metric, idx->w_lut.as<float>());
}

// K1f: the values of rows c0 .. c0 + nc for the qc queries whose tables are in w_lut -> w_vals (ld kFlatTile)
static void pq_flat_values(dfx_index* idx, int64_t qc, int64_t c0, int64_t nc, cudaStream_t st) {
    const int M = idx->M;
    const int64_t span = pq_flat_span(qc, nc);
    const unsigned grid = (unsigned)(qc * dfx_ceil_div(nc, span));
    const size_t smem = (size_t)M * PQF_KSUB * 4;
    pq_flat_dispatch(M, [&](auto MT, auto W) {
        auto kern = pq_flat_values_kernel<decltype(MT)::value, decltype(W)::value>;
        DFX_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        DFX_LAUNCH(kern, grid, PQF_THREADS, smem, st, idx->w_lut.as<float>(), idx->payload.as<uint8_t>(), c0, (int)nc,
                   (int)span, (int)qc, M, idx->w_vals.as<float>(), kFlatTile);
    });
}

// The values of a flat shard, shared by search and range search: per chunk of up to 1024 queries, each
// tile of up to kFlatTile columns goes to w_vals (ld kFlatTile, 128 MB at most), and tile(q0, qc, c0, nc)
// reads it before the next tile overwrites it.  FLAT / FLAT_SQ16: the FFMA GEMM (K1a) over the fp32 or
// fp16 rows; FLAT_PQ: the chunk's tables (K3f), then K1f over the codes.
template <class Tile>
static void flat_tiles(dfx_index* idx, int64_t nq, const float* d_x, cudaStream_t st, Tile&& tile) {
    const int d = idx->cfg.d;
    const int64_t N = idx->n_sorted;
    const bool pq = idx->cfg.kind == DFX_FLAT_PQ;
    const int64_t QC = std::min<int64_t>(nq, (32ll << 20) / kFlatTile);
    const float* xnorm = idx->xnorm.as<float>();
    idx->w_vals.reserve((size_t)QC * kFlatTile * 4);
    for (int64_t q0 = 0; q0 < nq; q0 += QC) {
        const int64_t qc = std::min(QC, nq - q0);
        if (pq) pq_flat_tables(idx, d_x + q0 * d, qc, st);
        for (int64_t c0 = 0; c0 < N; c0 += kFlatTile) {
            const int64_t nc = std::min(kFlatTile, N - c0);
            if (pq) {
                pq_flat_values(idx, qc, c0, nc, st);
            } else {
                dfx_with_flat_rows(idx, [&](auto rows) {
                    dfx_launch_gemm_values(d_x + q0 * d, qc, rows + c0 * d, xnorm ? xnorm + c0 : nullptr, nc, d,
                                           idx->cfg.metric, idx->w_vals.as<float>(), kFlatTile, st);
                });
            }
            tile(q0, qc, c0, nc);
        }
    }
}

// FLAT_PQ searches that take the fused per-tile top-k (K4f) instead of the values tiles (K1f).  Measured on an
// H100 at N = 10 M (DESIGN.md section 4.14): K4f is ahead at every nq for k <= 100, and at larger k while
// nq * k <= 16384; above that its per-warp queues of 2 next_pow2(k) composites and the chunk cap's re-reads of
// the codes cost more than writing and re-reading the values.
static bool pq_flat_fused(int64_t nq, int k) { return k <= 1024 && (k <= 100 || nq * k <= 16384); }

// FLAT_PQ, pq_flat_fused: per query chunk the tables (K3f), K4f over every row tile into the chunk's partial
// rows (ntiles * k composites per query), then the k best of each row.  The chunk keeps its partial rows
// within the 128 MiB the IVF path allows its partial results (a tile grows when one query alone would
// not fit).
static void search_flat_pq(dfx_index* idx, int64_t nq, const float* d_x, int k, float* d_D, int64_t* d_I,
                           cudaStream_t st) {
    const int d = idx->cfg.d, M = idx->M;
    const int64_t N = idx->n_sorted;
    const int64_t part_max = (int64_t)1 << 24;
    int64_t tile = pq_flat_span(std::min<int64_t>(nq, 1024), N);
    while (dfx_ceil_div(N, tile) * k > part_max) tile <<= 1;
    const int64_t ntiles = dfx_ceil_div(N, tile), ld = ntiles * k;
    const int64_t QC = std::max<int64_t>(1, std::min<int64_t>({nq, 1024, part_max / ld}));
    const int cap = 2 * dfx_next_pow2(k < 32 ? 32 : k);
    const size_t smem = (size_t)M * PQF_KSUB * 4 + dfx_scan_queue_smem(PQF_THREADS, cap, false);
    idx->w_part.reserve((size_t)QC * ld * 8);
    uint64_t* part = idx->w_part.as<uint64_t>();
    for (int64_t q0 = 0; q0 < nq; q0 += QC) {
        const int64_t qc = std::min(QC, nq - q0);
        pq_flat_tables(idx, d_x + q0 * d, qc, st);
        pq_flat_dispatch(M, [&](auto MT, auto W) {
            auto kern = pq_flat_topk_kernel<decltype(MT)::value, decltype(W)::value>;
            DFX_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
            DFX_LAUNCH(kern, (unsigned)(qc * ntiles), PQF_THREADS, smem, st, idx->w_lut.as<float>(),
                       idx->payload.as<uint8_t>(), N, tile, (int)qc, M, k, cap, part, ld);
        });
        ResultWriter wr{d_D + q0 * k, d_I + q0 * k, k, idx->cfg.metric, nullptr};
        dfx_launch_select<128>(CompLoader{part, ld}, wr, qc, (int)ld, k, st);
    }
}

static void search_flat(dfx_index* idx, int64_t nq, const float* d_x, int64_t k64, float* d_D, int64_t* d_I,
                        cudaStream_t st) {
    DFX_REQUIRE(k64 <= 4096, "flat search supports k <= 4096");
    const int d = idx->cfg.d;
    const int k = (int)k64;
    const int64_t N = idx->n_sorted;
    const int metric = idx->cfg.metric;
    if (N == 0) {
        ResultWriter wr{d_D, d_I, k, metric, nullptr};
        CompLoader ldr{nullptr, 0};
        dfx_launch_select<128>(ldr, wr, nq, 0, k, st);
        return;
    }
    if (idx->cfg.kind == DFX_FLAT_PQ && pq_flat_fused(nq, k)) return search_flat_pq(idx, nq, d_x, k, d_D, d_I, st);
    const float* qnorm = query_norms(idx, nq, d_x, idx->w_dis0, st);
    if (idx->flat_rows() && idx->flat_tc && idx->tc_enabled && dfx_tc_flat_covers(idx, k) &&
        dfx_tc_flat_table(idx, st)) {  // screening on tensor cores + exact re-rank
        const int64_t ng = dfx_ceil_div(N, 128) * 4;
        const int64_t QT = std::max<int64_t>(128, ((64ll << 20) / (ng * 4)) / 128 * 128);
        for (int64_t q0 = 0; q0 < nq; q0 += QT) {
            const int64_t qc = std::min(QT, nq - q0);
            const int ncand = dfx_tc_flat_candidates(idx, d_x + q0 * d, qc, k, st);
            CompLoader ldr{idx->tc_cand.as<uint64_t>(), ncand};
            ResultWriter wr{d_D + q0 * k, d_I + q0 * k, k, metric, qnorm ? qnorm + q0 : nullptr};
            dfx_launch_select<128>(ldr, wr, qc, ncand, k, st);
        }
        return;
    }
    // each tile's k best into the chunk's partial rows (slot t * k), then after a chunk's last tile the k
    // best of all its tiles
    const int64_t ntiles = dfx_ceil_div(N, kFlatTile);
    flat_tiles(idx, nq, d_x, st, [&](int64_t q0, int64_t qc, int64_t c0, int64_t nc) {
        idx->w_part.reserve((size_t)qc * ntiles * k * 8);
        uint64_t* part = idx->w_part.as<uint64_t>();
        dfx_launch_select_cols(idx->w_vals.as<float>(), qc, (int)nc, kFlatTile, k, (uint32_t)c0, nullptr, nullptr,
                               part + c0 / kFlatTile * k, ntiles * k, st);
        if (c0 + nc < N) return;
        ResultWriter wr{d_D + q0 * k, d_I + q0 * k, k, metric, qnorm ? qnorm + q0 : nullptr};
        dfx_launch_select<128>(CompLoader{part, ntiles * k}, wr, qc, (int)(ntiles * k), k, st);
    });
}

// the IVF list scans; plan_ivf picks one per search
enum class ScanFamily {
    Fs,      // IVF-PQ FastScan: u8 quantized table, integer sums (scan_pq_fs_kernel<M>)
    Pq4,     // IVF-PQ, 4-bit codes: table in registers (scan_pq4_kernel<M>)
    PqIl2,   // IVF-PQ, M = 32 interleaved: table build and block scan in one kernel (dfx_scan_il2.cu)
    PqWide,  // IVF-PQ, 64 < M <= 128: the scan builds the table in its own shared memory
    Pq,      // IVF-PQ, 8-bit row-major codes, M <= 64 (scan_pq_kernel)
    Rows,    // IVF-Flat, IVF-SQ fp16, IVF-SQ8 (scan_rows_kernel)
};

// what an IVF search decides once, before it launches anything
struct IvfPlan {
    int kind;            // the first stage's kind (IVF_PQR: IVF_PQ)
    bool refine, rflat;  // IVF-PQR or the flat refinement: k candidates re-ranked down to kout
    int k, kout;         // k = k' = k * k_factor when refining, else kout
    int nprobe;
    bool mat;            // k > 1024: candidate rows of ld slots instead of per-warp queues
    int64_t ld;
    int64_t QC;          // queries per chunk
    int cap;             // composites per warp queue: 2 KP, KP = next_pow2(max(k, 32))
    int wide_threads;    // PqWide: the CTA shape
    int smetric;         // the list scan's metric (the coarse quantizer's is cfg.metric)
    bool use_tc;         // coarse quantizer on tensor cores
    ScanFamily family;
};

// Every refusal of the IVF path is here, in this order, so a refused search launches nothing (the M
// checks of launch_list_scan only guard shapes dfx_create refuses).  Runs after the pending rows are
// finalized, which can change the layout (idx->il).  A range search (range, k64 = 1) takes the
// candidate rows whatever its radius.
static IvfPlan plan_ivf(dfx_index* idx, int64_t nq, int64_t k64, bool range = false) {
    IvfPlan p{};
    // IVF-PQR and the flat refinement: the base kind's search for k' = (int64)(k * k_factor)
    // candidates (faiss's float product) into workspace rows, re-ranked per query chunk down to
    // kout = k; every sizing rule below sees k'
    p.rflat = idx->rflat();
    p.refine = idx->cfg.kind == DFX_IVF_PQR || p.rflat;
    const int64_t kfirst = p.refine ? (int64_t)((float)k64 * idx->k_factor) : k64;
    p.kout = (int)k64;
    const int k = p.k = (int)std::min<int64_t>(kfirst, 1 << 30);
    p.kind = idx->cfg.kind == DFX_IVF_PQR ? DFX_IVF_PQ : idx->cfg.kind;
    if (p.kind == DFX_IVF_PQ_FS) p.family = ScanFamily::Fs;
    else if (p.kind != DFX_IVF_PQ) p.family = ScanFamily::Rows;
    else if (idx->ksub == 16) p.family = ScanFamily::Pq4;
    else if (idx->il) p.family = ScanFamily::PqIl2;
    else if (idx->M > 64) p.family = ScanFamily::PqWide;
    else p.family = ScanFamily::Pq;

    DFX_REQUIRE(k64 <= 4096, "IVF search supports k <= 4096");
    const int pqr_kmax = 16384;  // candidate rows selected by select_cand_kernel: P * 8 = 128 KiB of shared memory
    DFX_REQUIRE(!p.refine || kfirst <= pqr_kmax,
                std::string(p.rflat ? "RFlat" : "IVF-PQR") + " search at k=" + std::to_string(k64) +
                    " with k_factor=" + std::to_string(idx->k_factor) + ": k' = " + std::to_string(kfirst) + " candidates to re-rank, more than " +
                    std::to_string(pqr_kmax));
    const int64_t nlist = idx->cfg.nlist;
    const int nprobe = p.nprobe = (int)std::min<int64_t>(std::max<int64_t>(idx->nprobe, 1), nlist);
    DFX_REQUIRE(nprobe <= 4096, "nprobe <= 4096");
    p.mat = range || k > 1024;
    const int64_t part_max = (int64_t)1 << 24;  // composites of a chunk's partial results / candidates (128 MiB)
    if (p.mat) {
        DFX_REQUIRE(idx->h_len_top.size() == (size_t)nlist + 1, "IVF search: list lengths are not known");
        p.ld = std::max<int64_t>(idx->h_len_top[(size_t)nprobe], 1);
        DFX_REQUIRE(p.ld <= part_max,
                    (range ? std::string("IVF range search") : "IVF search at k=" + std::to_string(k)) +
                        " with nprobe=" + std::to_string(nprobe) +
                        ": one query's candidates can reach " + std::to_string(p.ld) +
                        " vectors (the nprobe longest lists), more than the 16777216 (128 MiB) of a query chunk");
    }
    p.smetric = (p.kind == DFX_IVF_FLAT) ? idx->cfg.metric : DFX_METRIC_L2;

    // query chunk: bounds the workspace (values matrix on the FFMA coarse path, tables and
    // partial results otherwise)
    p.use_tc = idx->tc_enabled && idx->tc_ready && nlist >= 1024 && nprobe <= 512;
    int64_t QC = p.use_tc ? 8192 : (32ll << 20) / nlist;
    if (QC < 1) QC = 1;
    if (QC > 8192) QC = 8192;
    // the chunk's partial results (qc x ngroups x k composites) stay within the values matrix's
    // 128 MiB: cap QC against ngroups <= nprobe, then once more against the ngroups choose_group
    // gives at that cap (choose_group never gives a larger chunk more groups per query).
    // k > 1024: the chunk's candidate rows (qc x ld composites) stay within the same 128 MiB.
    const int64_t q1 = std::max<int64_t>(1, part_max / ((int64_t)nprobe * k));
    if (p.mat) {
        QC = std::min(QC, part_max / p.ld);
    } else if (QC > q1) {
        const int G1 = choose_group(q1, nprobe);
        const int64_t ng1 = (nprobe + G1 - 1) / G1;
        QC = std::min(QC, std::max(q1, part_max / (ng1 * k)));
    }
    // refinements: the chunk's first-stage rows and refined composites (qc x k' of each) stay within 2^22
    const int64_t pqr_cand_max = (int64_t)1 << 22;
    if (p.refine) QC = std::min(QC, std::max<int64_t>(1, pqr_cand_max / k));
    if (QC > nq) QC = nq;
    p.QC = QC;
    p.cap = 2 * dfx_next_pow2(k < 32 ? 32 : k);

    // 64 < M <= 128: the widest CTA whose table and per-warp queues fit in the device's shared memory
    // (k > 1024: no queues, the table alone; the 512-thread shape, the only one instantiated)
    if (p.family == ScanFamily::PqWide) {
        const size_t optin = (size_t)dfx_smem_optin();
        for (int t : {512, 256, 128}) {
            if (dfx_pq_wide_smem(idx->M, t, p.cap, p.mat) <= optin) {
                p.wide_threads = t;
                break;
            }
        }
        DFX_REQUIRE(!p.mat || p.wide_threads == 512, "IVF-PQ with " + std::to_string(idx->M) +
                                                         " sub-quantizers: the table does not fit in shared memory");
        DFX_REQUIRE(p.wide_threads > 0,
                    "IVF-PQ with " + std::to_string(idx->M) + " sub-quantizers at k=" + std::to_string(k) +
                        ": the distance table and the candidate queues need " +
                        std::to_string(dfx_pq_wide_smem(idx->M, 128, p.cap, p.mat)) +
                        " bytes of shared memory per thread block, the device allows " + std::to_string(optin));
    }
    DFX_REQUIRE(!p.refine || p.rflat || idx->inv_valid, "IVF-PQR search: the id -> position map is not built");
    return p;
}

// M of the 4-bit and FastScan scans: a multiple of 8 in [8, 128] (checked by dfx_create)
using PqMByEight = IntList<8, 16, 24, 32, 40, 48, 56, 64, 72, 80, 88, 96, 104, 112, 120, 128>;

// a list-scan launch, opted in to its dynamic shared memory
template <class K, class... A>
static void launch_scan(K kern, unsigned grid, int threads, size_t smem, cudaStream_t st, A... args) {
    DFX_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    DFX_LAUNCH(kern, grid, threads, smem, st, args...);
}

// K3 + K4: the list scan of one query chunk, with the table its family needs.  It writes per-group
// partial results or, k > 1024, the candidate rows into `part`; returns true when it wrote the
// chunk's final rows (outD, outI) itself.
static bool launch_list_scan(dfx_index* idx, const IvfPlan& p, const float* xq, int64_t qc, const int32_t* keys,
                             int G, int ngroups, uint64_t* part, const int64_t* coff, float* outD, int64_t* outI,
                             cudaStream_t st) {
    const int d = idx->cfg.d, M = idx->M, ksub = idx->ksub, k = p.k, cap = p.cap, nprobe = p.nprobe;
    const unsigned grid = (unsigned)(qc * ngroups);
    const size_t queues = dfx_scan_queue_smem(128, cap, p.mat);  // the 128-thread scans' candidate queues
    if (p.family == ScanFamily::Pq || p.family == ScanFamily::PqWide || p.family == ScanFamily::Pq4) {
        // K3: each query's [M][ksub] table (w_lut; the wide scan builds its own) and the exact
        // |q - c|^2 of its probed lists (w_dis0)
        const bool lut = p.family != ScanFamily::PqWide;
        if (lut) idx->w_lut.reserve((size_t)qc * M * ksub * 4);
        idx->w_dis0.reserve((size_t)qc * nprobe * 4);
        DFX_LAUNCH(pq_prep_kernel, (unsigned)qc, 256, (size_t)((d + 3) / 4) * 16, st, xq, d, M, ksub, idx->dsub,
                   idx->codebooks.as<float>(), idx->centroids.as<float>(), keys, nprobe,
                   lut ? idx->w_lut.as<float>() : nullptr, idx->w_dis0.as<float>());
    }
    switch (p.family) {
        case ScanFamily::Fs: {
            // each query's table quantized to u8 (w_lut) with its (1 / a, b) (w_dis0), then the
            // integer scan; fs_dequant_kernel maps the selected distances after the selection
            idx->w_lut.reserve((size_t)qc * M * 16);
            idx->w_dis0.reserve((size_t)qc * 8);
            DFX_LAUNCH(pq_fs_lut_kernel, (unsigned)qc, 256, dfx_pq_fs_lut_smem(d, M), st, xq, d, M, idx->dsub,
                       idx->codebooks.as<float>(), idx->w_lut.as<uint8_t>(), idx->w_dis0.as<float2>());
            const bool found = dispatch_int(PqMByEight{}, M, [&](auto MT) {
                launch_scan(p.mat ? scan_pq_fs_kernel<MT, true> : scan_pq_fs_kernel<MT>, grid, 128, queues, st,
                            idx->w_lut.as<uint8_t>(), keys, nprobe, G, ngroups, idx->list_off.as<int64_t>(),
                            idx->payload.as<uint8_t>(), idx->ids.as<int32_t>(), k, cap, part, coff);
            });
            DFX_REQUIRE(found, "IVF-PQ FastScan: no list scan for M=" + std::to_string(M));
            return false;
        }
        case ScanFamily::Pq4: {
            const bool found = dispatch_int(PqMByEight{}, M, [&](auto MT) {
                launch_scan(p.mat ? scan_pq4_kernel<MT, true> : scan_pq4_kernel<MT>, grid, 128, queues, st,
                            idx->w_lut.as<float>(), idx->w_dis0.as<float>(), keys, nprobe, G, ngroups,
                            idx->list_off.as<int64_t>(), idx->payload.as<uint8_t>(), idx->tvals.as<float>(),
                            idx->ids.as<int32_t>(), k, cap, part, coff);
            });
            DFX_REQUIRE(found, "IVF-PQ with 4-bit codes: no list scan for M=" + std::to_string(M));
            return false;
        }
        case ScanFamily::PqIl2:
            // with a single probe group per query the scan also writes the final rows
            if (!p.mat) return dfx_launch_scan_pq_il2(idx, xq, qc, keys, nprobe, G, ngroups, k, cap, part, outD, outI, st);
            dfx_launch_scan_pq_il2_mat(idx, xq, qc, keys, nprobe, G, ngroups, part, coff, st);
            return false;
        case ScanFamily::PqWide: {
            const size_t smem = dfx_pq_wide_smem(M, p.wide_threads, cap, p.mat);
            const int mt = (M == 128 || M == 96) ? M : 0;  // any other M % 4 == 0: 32-bit code loads
            // M = 96 never takes 128 threads on a device that opts in to 232448 B (sm_90): at 256
            // threads the largest queues (k <= 1024, cap = 2048) take 96 KB of table + 8 warps x 2048
            // x 8 B = 229376 B.  So <96, 128> is not instantiated; a device that offers less is refused.
            bool found = false;
            dispatch_int(IntList<128, 96, 0>{}, mt, [&](auto MT) {
                const auto launch = [&](auto THREADS) {
                    launch_scan(p.mat ? scan_pq_wide_kernel<MT, 512, true> : scan_pq_wide_kernel<MT, THREADS>, grid,
                                p.wide_threads, smem, st, xq, d, M, idx->dsub, idx->codebooks.as<float>(),
                                idx->w_dis0.as<float>(), keys, nprobe, G, ngroups, idx->list_off.as<int64_t>(),
                                idx->payload.as<uint8_t>(), idx->tvals.as<float>(), idx->ids.as<int32_t>(), k, cap,
                                part, coff);
                };
                if constexpr (MT == 96) found = dispatch_int(IntList<512, 256>{}, p.wide_threads, launch);
                else found = dispatch_int(IntList<512, 256, 128>{}, p.wide_threads, launch);
            });
            DFX_REQUIRE(found, "IVF-PQ with " + std::to_string(M) + " sub-quantizers: no list scan of " +
                                   std::to_string(p.wide_threads) + " threads");
            return false;
        }
        case ScanFamily::Pq: {
            const size_t smem = (size_t)M * ksub * 4 + queues;
            const int mt = (M == 8 || M == 16 || M == 32 || M == 64) ? M : 0;  // other M: padded to 64 with +0
            dispatch_int(IntList<8, 16, 32, 64, 0>{}, mt, [&](auto MT) {
                launch_scan(p.mat ? scan_pq_kernel<MT, true> : scan_pq_kernel<MT>, grid, 128, smem, st,
                            idx->w_lut.as<float>(), idx->w_dis0.as<float>(), keys, nprobe, G, ngroups,
                            idx->list_off.as<int64_t>(), idx->payload.as<uint8_t>(), idx->tvals.as<float>(),
                            idx->ids.as<int32_t>(), M, ksub, k, cap, part, coff);
            });
            return false;
        }
        case ScanFamily::Rows: {
            // shared memory: the query; + the raw query (SQ16); + vmin and vdiff (SQ8)
            const int dq = (p.kind == DFX_IVF_SQ8) ? 4 * d : (p.kind == DFX_IVF_SQ16) ? 2 * d : d;
            const size_t smem = (((size_t)dq * 4 + 15) / 16) * 16 + queues;
            // vectors in flight per warp: rows of up to 1 KB need 8 to cover the DRAM latency,
            // longer rows keep 4 (rows_inflight overrides)
            const int inflight = idx->rows_inflight ? idx->rows_inflight : (idx->row_bytes() <= 1024 ? 8 : 4);
            const int mode = p.kind == DFX_IVF_SQ8 ? 3 : p.kind == DFX_IVF_SQ16 ? 2 : p.smetric == DFX_METRIC_IP ? 0 : 1;
            dispatch_int(IntList<0, 1, 2, 3>{}, mode, [&](auto MODE) {
                dispatch_int(IntList<4, 8>{}, inflight, [&](auto U) {
                    launch_scan(p.mat ? scan_rows_kernel<MODE, U, true> : scan_rows_kernel<MODE, U>, grid, 128, smem,
                                st, xq, d, idx->centroids.as<float>(), keys, nprobe, G, ngroups,
                                idx->list_off.as<int64_t>(), idx->payload.p, idx->ids.as<int32_t>(), k, cap, part,
                                idx->sq_trained.as<float>(), coff);
                });
            });
            return false;
        }
    }
    return false;
}

// K1: the nprobe lists each query of a chunk probes -- tensor cores (screen) + canonical fp32
// (decide), or plain FFMA
static void coarse_probes(dfx_index* idx, const IvfPlan& p, const float* xq, int64_t qc, int32_t* keys,
                          cudaStream_t st) {
    const int64_t nlist = idx->cfg.nlist;
    if (p.use_tc) {
        dfx_tc_coarse_search(idx, xq, qc, p.nprobe, keys, st);
    } else {
        idx->w_vals.reserve((size_t)p.QC * nlist * 4);
        dfx_launch_gemm_values(xq, qc, idx->centroids.as<float>(), idx->cnorm.as<float>(), nlist, idx->cfg.d,
                               idx->cfg.metric, idx->w_vals.as<float>(), nlist, st);
        dfx_launch_select_cols(idx->w_vals.as<float>(), qc, (int)nlist, nlist, p.nprobe, 0, keys, nullptr, nullptr,
                               0, st);
    }
}

// what the list scan of one query chunk leaves for the caller
struct IvfChunk {
    int64_t q0, qc;
    const float* xq;       // the chunk's queries
    uint64_t* part;        // the per-group partial results or, p.mat, the candidate rows
    int64_t* coff;         // p.mat: [qc][nprobe + 1] slot offsets of the candidate rows
    int ngroups;
    float* outD;           // where the selection writes: the result rows, or (refinements) the first-stage rows
    int64_t* outI;
    bool final_written;    // the scan wrote outD, outI itself
};

// The query chunks of an IVF search or range search: per chunk of p.QC queries, its probes (K1), with
// p.mat the slot offsets of its candidate rows (K_off), and its list scan (K3 + K4, the profiled scan
// range); then chunk(c) takes what the scan left.  The probes of every query stay in w_keys for
// dfx_last_stats.  A range search passes no result rows (d_D, d_I null).
template <class Chunk>
static void ivf_chunks(dfx_index* idx, const IvfPlan& p, int64_t nq, const float* d_x, float* d_D, int64_t* d_I,
                       cudaStream_t st, Chunk&& chunk) {
    const int d = idx->cfg.d, k = p.k, nprobe = p.nprobe;
    idx->w_keys.reserve((size_t)nq * nprobe * 4);
    if (p.mat) idx->w_coff.reserve((size_t)p.QC * (nprobe + 1) * 8);
    if (p.refine) {
        idx->w_rD.reserve((size_t)p.QC * k * 4);
        idx->w_rI.reserve((size_t)p.QC * k * 8);
        idx->w_rcomp.reserve((size_t)p.QC * k * 8);
    }
    IvfChunk c{};
    c.coff = p.mat ? idx->w_coff.as<int64_t>() : nullptr;
    for (c.q0 = 0; c.q0 < nq; c.q0 += p.QC) {
        c.qc = std::min(p.QC, nq - c.q0);
        c.xq = d_x + c.q0 * d;
        c.outD = p.refine ? idx->w_rD.as<float>() : d_D ? d_D + c.q0 * k : nullptr;
        c.outI = p.refine ? idx->w_rI.as<int64_t>() : d_I ? d_I + c.q0 * k : nullptr;
        int32_t* keys = idx->w_keys.as<int32_t>() + c.q0 * nprobe;
        coarse_probes(idx, p, c.xq, c.qc, keys, st);
        const int G = choose_group(c.qc, nprobe);
        c.ngroups = (nprobe + G - 1) / G;
        idx->w_part.reserve(p.mat ? (size_t)c.qc * p.ld * 8 : (size_t)c.qc * c.ngroups * k * 8);
        c.part = idx->w_part.as<uint64_t>();
        if (p.mat)
            DFX_LAUNCH(cand_offsets_kernel, (unsigned)dfx_ceil_div(c.qc, 4), 128, 0, st, keys, c.qc, nprobe,
                       idx->list_off.as<int64_t>(), p.ld, c.coff);
        if (idx->prof_on) idx->prof_scan.begin(st);
        c.final_written = launch_list_scan(idx, p, c.xq, c.qc, keys, G, c.ngroups, c.part, c.coff, c.outD, c.outI, st);
        if (idx->prof_on) idx->prof_scan.end(st);
        chunk(c);
    }
    idx->last_nq = nq;
    idx->last_nprobe = nprobe;
    idx->last_keys_valid = true;
}

// What every search and range search does first: the statistics of the last search and the results of
// the last range search stop being valid, and rows added since the last call join the lists.
static void begin_query(dfx_index* idx, cudaStream_t st) {
    idx->last_keys_valid = false;
    idx->r_total = -1;
    if (idx->n_pending > 0) dfx_finalize_impl(idx, st);
}

void dfx_search_impl(dfx_index* idx, int64_t nq, const float* d_x, int64_t k64, float* d_D,
                     int64_t* d_I, cudaStream_t st) {
    DFX_REQUIRE(idx->trained || idx->flat_rows(), "index is not trained");
    DFX_REQUIRE(k64 >= 1, "k must be >= 1");
    if (nq <= 0) return;
    begin_query(idx, st);
    if (idx->is_flat()) return search_flat(idx, nq, d_x, k64, d_D, d_I, st);

    const IvfPlan p = plan_ivf(idx, nq, k64);
    const int k = p.k, kout = p.kout;
    ivf_chunks(idx, p, nq, d_x, d_D, d_I, st, [&](const IvfChunk& c) {
        ResultWriter wr{c.outD, c.outI, k, p.smetric, nullptr};
        if (p.mat) {
            // P >= 2048 = sort_cap: a row of up to sort_cap candidates is sorted whole
            const int P = dfx_next_pow2(k);
            if ((size_t)P * 8 > 48 * 1024)  // a refinement's k' > 4096: opt in to more shared memory
                DFX_CUDA(cudaFuncSetAttribute(select_cand_kernel<256>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                              P * 8));
            DFX_LAUNCH(select_cand_kernel<256>, (unsigned)c.qc, 256, (size_t)P * 8, st, c.part, c.coff, p.nprobe, wr,
                       k, P, 2048);
        } else if (!c.final_written) {
            dfx_launch_select<128>(CompLoader{c.part, (int64_t)c.ngroups * k}, wr, c.qc, c.ngroups * k, k, st);
        }
        if (p.family == ScanFamily::Fs && !p.rflat)  // the flat refinement reads the first stage's ids only
            DFX_LAUNCH(fs_dequant_kernel, (unsigned)dfx_ceil_div(c.qc * k, 256), 256, 0, st, c.outD, c.outI,
                       c.qc * k, k, idx->w_dis0.as<float2>());
        if (p.refine)
            refine_candidates(idx, c.xq, c.qc, k, kout, c.outI, d_D + c.q0 * kout, d_I + c.q0 * kout, st);
    });
}

// =====================================================================================
// Range search: every vector a search of the same shard scores whose distance passes the radius
// (L2: D < radius, IP: D > radius, strict as in faiss; NaN never passes), with the distances the
// k-NN search reports.  FLAT calls flat_tiles, IVF calls ivf_chunks with the candidate rows of k > 1024
// (plan_ivf in range mode).  Each piece -- FLAT: one column tile of a query chunk, IVF: one
// query chunk -- is counted per query (K_rc), scanned, read back (8 bytes, so the result buffers
// grow to fit and the 2^27 limit is enforced before anything is written) and its passing composites
// appended query by query (K_re).  Then each query's results are made contiguous (FLAT with several
// tiles: a stable sort by query) and sorted by composite: segments of up to 2048 in shared memory
// (K_rs), or, when one is longer, two stable device-wide sorts (by composite, then by query).
// =====================================================================================
static constexpr int64_t kRangeMaxResults = (int64_t)1 << 27;  // per call and shard (1.5 GiB of results)
static constexpr int kRangeSortCap = 2048;

__device__ __forceinline__ bool dfx_range_pass(float v, int metric, float radius) {
    return metric == DFX_METRIC_IP ? v > radius : v < radius;
}

struct RangeCandRows {  // IVF: query q's candidate row of a chunk
    const uint64_t* part;
    const int64_t* coff;
    int nprobe;
    __device__ __forceinline__ int64_t start(int64_t q) const { return coff[q * (nprobe + 1)]; }
    __device__ __forceinline__ int64_t size(int64_t q) const { return coff[q * (nprobe + 1) + nprobe] - start(q); }
    __device__ __forceinline__ uint64_t comp(int64_t s, int64_t e) const { return part[s + e]; }
};
struct RangeTileRows {  // FLAT: query q's row of a values tile of nc columns from column c0
    const float* vals;
    int64_t ld, nc;
    uint32_t c0;
    __device__ __forceinline__ int64_t start(int64_t q) const { return q * ld; }
    __device__ __forceinline__ int64_t size(int64_t) const { return nc; }
    __device__ __forceinline__ uint64_t comp(int64_t s, int64_t e) const {
        return dfx_comp(vals[s + e], c0 + (uint32_t)e);
    }
};

// K_rc: one warp per query, cnt[q] = the entries of its row that pass
template <class Rows>
__global__ void __launch_bounds__(128)
range_count_kernel(Rows rows, int64_t nq, int metric, const float* __restrict__ qnorm, float radius,
                   int64_t* __restrict__ cnt) {
    const int64_t q = (int64_t)blockIdx.x * 4 + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (q >= nq) return;  // warp-uniform
    const int64_t s = rows.start(q), n = rows.size(q);
    long long c = 0;
    for (int64_t e0 = 0; e0 < n; e0 += 32) {
        const int64_t e = e0 + lane;
        const bool pass = e < n && dfx_range_pass(dfx_result_distance(rows.comp(s, e), metric, qnorm, q), metric, radius);
        c += __popc(__ballot_sync(0xffffffffu, pass));
    }
    if (lane == 0) cnt[q] = c;
}

// K_re: the same walk; the passing composites of query q go to out[off[q] ..] in row order (ballot
// prefix) with their query q0 + q, and tot[q0 + q] adds them to the query's results of the call
template <class Rows>
__global__ void __launch_bounds__(128)
range_emit_kernel(Rows rows, int64_t nq, int metric, const float* __restrict__ qnorm, float radius,
                  const int64_t* __restrict__ off, int64_t q0, uint64_t* __restrict__ out, uint32_t* __restrict__ qout,
                  int64_t* __restrict__ tot) {
    const int64_t q = (int64_t)blockIdx.x * 4 + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (q >= nq) return;  // warp-uniform
    const int64_t s = rows.start(q), n = rows.size(q);
    int64_t pos = off[q];
    for (int64_t e0 = 0; e0 < n; e0 += 32) {
        const int64_t e = e0 + lane;
        uint64_t c = DFX_COMP_NONE;
        bool pass = false;
        if (e < n) {
            c = rows.comp(s, e);
            pass = dfx_range_pass(dfx_result_distance(c, metric, qnorm, q), metric, radius);
        }
        const unsigned m = __ballot_sync(0xffffffffu, pass);
        if (pass) {
            const int64_t i = pos + __popc(m & ((1u << lane) - 1u));
            out[i] = c;
            qout[i] = (uint32_t)(q0 + q);
        }
        pos += __popc(m);
    }
    if (lane == 0) tot[q0 + q] += off[q + 1] - off[q];
}

// K_rs: one CTA per query sorts its contiguous segment of at most kRangeSortCap composites
__global__ void __launch_bounds__(256) range_sort_kernel(const int64_t* __restrict__ lims, uint64_t* __restrict__ comp) {
    DFX_DYN_SMEM(unsigned char, smem_raw, 16);
    uint64_t* s = reinterpret_cast<uint64_t*>(smem_raw);
    const int64_t b = lims[blockIdx.x];
    const int n = (int)(lims[blockIdx.x + 1] - b);
    if (n < 2) return;  // CTA-uniform
    int P = 2;
    while (P < n) P <<= 1;
    for (int e = threadIdx.x; e < P; e += 256) s[e] = e < n ? comp[b + e] : DFX_COMP_NONE;
    dfx_block_bitonic_sort<256>(s, P);
    for (int e = threadIdx.x; e < n; e += 256) comp[b + e] = s[e];
}

// K_rm: composites -> (D, I), the mapping of ResultWriter
__global__ void range_map_kernel(const uint64_t* __restrict__ comp, const uint32_t* __restrict__ qidx, int64_t n,
                                 int metric, const float* __restrict__ qnorm, float* __restrict__ D,
                                 int64_t* __restrict__ I) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint64_t c = comp[i];
    D[i] = dfx_result_distance(c, metric, qnorm, qidx[i]);
    I[i] = (int64_t)(uint32_t)c;
}

// grow a result buffer of `elem`-byte entries to hold `need`, keeping its first `keep` entries
static void range_grow(DevBuf& b, int64_t need, int64_t keep, size_t elem, cudaStream_t st) {
    if ((size_t)need * elem <= b.cap) return;
    const int64_t n = std::min(kRangeMaxResults, std::max<int64_t>(need, (int64_t)(b.cap / elem) * 2));
    b.reserve((size_t)n * elem, (size_t)keep * elem, st);
}

// one piece of qc queries from query q0: count, scan, read back, check the limit, grow, emit
template <class Rows>
static void range_piece(dfx_index* idx, const Rows& rows, int64_t q0, int64_t qc, int metric, const float* qnorm,
                        float radius, int64_t& total, cudaStream_t st) {
    idx->r_cnt.reserve((size_t)(qc + 1) * 8);
    idx->r_off.reserve((size_t)(qc + 1) * 8);
    int64_t* cnt = idx->r_cnt.as<int64_t>();
    int64_t* off = idx->r_off.as<int64_t>();
    const unsigned grid = (unsigned)dfx_ceil_div(qc, 4);
    DFX_CUDA(cudaMemsetAsync(cnt + qc, 0, 8, st));
    DFX_LAUNCH(range_count_kernel<Rows>, grid, 128, 0, st, rows, qc, metric, qnorm, radius, cnt);
    size_t tb = 0;
    DFX_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, tb, cnt, off, (int)(qc + 1), st));
    idx->r_tmp.reserve(std::max<size_t>(tb, 16));
    DFX_CUDA(cub::DeviceScan::ExclusiveSum(idx->r_tmp.p, tb, cnt, off, (int)(qc + 1), st));
    int64_t n = 0;
    DFX_CUDA(cudaMemcpyAsync(&n, off + qc, 8, cudaMemcpyDeviceToHost, st));
    DFX_CUDA(cudaStreamSynchronize(st));
    DFX_REQUIRE(total + n <= kRangeMaxResults,
                "range search: the results of this call exceed 134217728 (2^27) on one shard; split the query batch");
    range_grow(idx->r_comp, total + n, total, 8, st);
    range_grow(idx->r_qidx, total + n, total, 4, st);
    DFX_LAUNCH(range_emit_kernel<Rows>, grid, 128, 0, st, rows, qc, metric, qnorm, radius, off, q0,
               idx->r_comp.as<uint64_t>() + total, idx->r_qidx.as<uint32_t>() + total, idx->r_tot.as<int64_t>());
    total += n;
}

// stable sort of n (key, value) pairs of the result buffers by key bits [0, bits), into the spare buffers,
// which then become the result buffers
template <class K, class V>
static void range_sort_pairs(dfx_index* idx, DevBuf& keys, DevBuf& keys2, DevBuf& vals, DevBuf& vals2, int64_t n,
                             int bits, cudaStream_t st) {
    keys2.reserve((size_t)n * sizeof(K));
    vals2.reserve((size_t)n * sizeof(V));
    size_t tb = 0;
    DFX_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, tb, keys.as<K>(), keys2.as<K>(), vals.as<V>(), vals2.as<V>(),
                                             (int)n, 0, bits, st));
    idx->r_tmp.reserve(std::max<size_t>(tb, 16));
    DFX_CUDA(cub::DeviceRadixSort::SortPairs(idx->r_tmp.p, tb, keys.as<K>(), keys2.as<K>(), vals.as<V>(),
                                             vals2.as<V>(), (int)n, 0, bits, st));
    std::swap(keys, keys2);
    std::swap(vals, vals2);
}

void dfx_range_impl(dfx_index* idx, int64_t nq, const float* d_x, float radius, int64_t* d_lims, int64_t* total_out,
                    cudaStream_t st) {
    // every refusal before anything is launched
    const int kind = idx->cfg.kind;
    DFX_REQUIRE(idx->trained || idx->flat_rows(), "index is not trained");
    DFX_REQUIRE(!std::isnan(radius), "range search: the radius is NaN");
    DFX_REQUIRE(kind != DFX_IVF_PQ_FS,
                "range search is not supported for IVF_PQ_FS (IVF-PQ FastScan) shards: their distances are "
                "dequantized only after the selection");
    DFX_REQUIRE(kind != DFX_IVF_PQR,
                "range search is not supported for IVF_PQR (refined IVF-PQ) shards: a radius over two stages of "
                "distances is not defined");
    DFX_REQUIRE(!idx->rflat(),
                "range search is not supported for shards with a flat refinement (refine_flat, \",RFlat\"): a "
                "radius over two stages of distances is not defined");
    DFX_REQUIRE(nq >= 0, "nq must be >= 0");
    if (nq == 0) {  // no results, and nothing to finalize
        idx->r_total = *total_out = 0;
        DFX_CUDA(cudaMemsetAsync(d_lims, 0, 8, st));
        return;
    }
    begin_query(idx, st);
    idx->r_tot.reserve((size_t)(nq + 1) * 8);
    int64_t* tot = idx->r_tot.as<int64_t>();
    DFX_CUDA(cudaMemsetAsync(tot, 0, (size_t)(nq + 1) * 8, st));
    int64_t total = 0;
    int metric = idx->cfg.metric;
    const float* qnorm = nullptr;
    bool grouped = true;  // the pieces left each query's results contiguous
    if (idx->is_flat()) {
        qnorm = query_norms(idx, nq, d_x, idx->r_qn, st);  // dfx_range_fetch_impl reads r_qn
        grouped = idx->n_sorted <= kFlatTile;
        flat_tiles(idx, nq, d_x, st, [&](int64_t q0, int64_t qc, int64_t c0, int64_t nc) {
            range_piece(idx, RangeTileRows{idx->w_vals.as<float>(), kFlatTile, nc, (uint32_t)c0}, q0, qc, metric,
                        qnorm ? qnorm + q0 : nullptr, radius, total, st);
        });
    } else {
        const IvfPlan p = plan_ivf(idx, nq, 1, true);
        metric = p.smetric;
        ivf_chunks(idx, p, nq, d_x, nullptr, nullptr, st, [&](const IvfChunk& c) {
            range_piece(idx, RangeCandRows{c.part, c.coff, p.nprobe}, c.q0, c.qc, metric, nullptr, radius, total, st);
        });
    }

    // lims = the exclusive scan of the per-query totals (tot[nq] = 0); the longest segment picks the sort
    size_t tb = 0;
    DFX_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, tb, tot, d_lims, (int)(nq + 1), st));
    idx->r_tmp.reserve(std::max<size_t>(tb, 16));
    DFX_CUDA(cub::DeviceScan::ExclusiveSum(idx->r_tmp.p, tb, tot, d_lims, (int)(nq + 1), st));
    std::vector<int64_t> lims((size_t)nq + 1);
    DFX_CUDA(cudaMemcpyAsync(lims.data(), d_lims, (size_t)(nq + 1) * 8, cudaMemcpyDeviceToHost, st));
    DFX_CUDA(cudaStreamSynchronize(st));
    int64_t longest = 0;
    for (int64_t q = 0; q < nq; q++) longest = std::max(longest, lims[(size_t)q + 1] - lims[(size_t)q]);
    int qbits = 1;  // the query index fits in qbits bits
    while (qbits < 32 && (1ll << qbits) < nq) qbits++;
    if (longest > kRangeSortCap) {
        range_sort_pairs<uint64_t, uint32_t>(idx, idx->r_comp, idx->r_comp2, idx->r_qidx, idx->r_qidx2, total, 64, st);
        range_sort_pairs<uint32_t, uint64_t>(idx, idx->r_qidx, idx->r_qidx2, idx->r_comp, idx->r_comp2, total, qbits,
                                             st);
    } else {
        // the pieces of several tiles interleave the queries: regroup even when no query holds more than one
        // result, or lims would hand one query's results to another
        if (!grouped && total > 1)
            range_sort_pairs<uint32_t, uint64_t>(idx, idx->r_qidx, idx->r_qidx2, idx->r_comp, idx->r_comp2, total,
                                                 qbits, st);
        if (longest > 1) {
            const int P = dfx_next_pow2((int)longest);
            DFX_LAUNCH(range_sort_kernel, (unsigned)nq, 256, (size_t)P * 8, st, d_lims, idx->r_comp.as<uint64_t>());
        }
    }
    idx->r_metric = metric;
    idx->r_qnorm = qnorm != nullptr;
    idx->r_total = *total_out = total;
}

void dfx_range_fetch_impl(dfx_index* idx, float* d_D, int64_t* d_I, cudaStream_t st) {
    DFX_REQUIRE(idx->r_total >= 0, "range fetch: no range search results (none ran, or a search ran since)");
    if (idx->r_total == 0) return;
    DFX_LAUNCH(range_map_kernel, (unsigned)dfx_ceil_div(idx->r_total, 256), 256, 0, st, idx->r_comp.as<uint64_t>(),
               idx->r_qidx.as<uint32_t>(), idx->r_total, idx->r_metric,
               idx->r_qnorm ? idx->r_qn.as<float>() : nullptr, d_D, d_I);
}

// ---- the cross-shard range merge (dfx_range_merge_dev).  S shards' range results, concatenated
// shard-major: shard s's query q holds entries base[s] + lims[s][q] .. base[s] + lims[s][q + 1] - 1,
// with base[s] = the totals lims[s'][nq] of the shards s' < s.  The merged order is the one of a stable
// sort by (query, score) over that concatenation, scores compared as floats (L2 ascending, IP
// descending): per query best first, equal scores by shard, then by the shard's own order.  Each run
// (one shard, one query) is already sorted that way, so every entry's output slot follows from ranks
// alone (co-ranking): the query's merged offset, the entry's rank r in its own run, and per other shard
// s' the entries of run (s', q) that precede it -- not worse than it when s' < s, strictly better when
// s' > s -- found by a binary search.  No atomics, no sort, deterministic.
// K_rml: one CTA; out_lims = exclusive scan over the queries of the summed run lengths
__global__ void __launch_bounds__(256)
range_merge_lims_kernel(int64_t S, int64_t nq, const int64_t* __restrict__ lims, int64_t* __restrict__ out_lims) {
    __shared__ long long s[256];
    long long carry = 0;
    for (int64_t q0 = 0; q0 < nq; q0 += 256) {
        const int64_t q = q0 + threadIdx.x;
        long long c = 0;
        if (q < nq)
            for (int64_t sh = 0; sh < S; sh++) c += lims[sh * (nq + 1) + q + 1] - lims[sh * (nq + 1) + q];
        s[threadIdx.x] = c;
        __syncthreads();
        for (int off = 1; off < 256; off <<= 1) {  // inclusive scan, Hillis-Steele
            const long long o = threadIdx.x >= off ? s[threadIdx.x - off] : 0;
            __syncthreads();
            s[threadIdx.x] += o;
            __syncthreads();
        }
        if (q < nq) out_lims[q] = carry + s[threadIdx.x] - c;
        carry += s[255];
        __syncthreads();
    }
    if (threadIdx.x == 0) out_lims[nq] = carry;
}

// entries of the sorted run x[0, n) that precede a value v: not worse (ties included) or strictly better
__device__ __forceinline__ int64_t range_merge_rank(const float* __restrict__ x, int64_t n, float v, bool maximize,
                                                    bool ties) {
    int64_t lo = 0, hi = n;
    while (lo < hi) {
        const int64_t mid = lo + ((hi - lo) >> 1);
        const float e = x[mid];
        const bool before = maximize ? (ties ? e >= v : e > v) : (ties ? e <= v : e < v);
        if (before) lo = mid + 1;
        else hi = mid;
    }
    return lo;
}

// K_rmm: one thread per entry i of the concatenation: its slot, then D, the payload and order[slot] = i
__global__ void __launch_bounds__(256)
range_merge_kernel(int64_t S, int64_t nq, int64_t T, const int64_t* __restrict__ lims, const float* __restrict__ D,
                   const int64_t* __restrict__ P, int maximize, const int64_t* __restrict__ out_lims,
                   float* __restrict__ outD, int64_t* __restrict__ outP, int64_t* __restrict__ order) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= T) return;
    // the shard: the last s whose base is <= i
    int64_t s = 0, base = 0;
    for (;;) {
        const int64_t tot = lims[s * (nq + 1) + nq];
        if (i < base + tot || s == S - 1) break;
        base += tot;
        s++;
    }
    // the query: the last q with lims[s][q] <= i - base
    const int64_t* L = lims + s * (nq + 1);
    const int64_t loc = i - base;
    int64_t lo = 0, hi = nq;  // lims[s][lo] <= loc < lims[s][hi]
    while (hi - lo > 1) {
        const int64_t mid = (lo + hi) >> 1;
        if (L[mid] <= loc) lo = mid;
        else hi = mid;
    }
    const int64_t q = lo;
    const float v = D[i];
    int64_t slot = out_lims[q] + (loc - L[q]);
    int64_t b2 = 0;
    for (int64_t s2 = 0; s2 < S; s2++) {
        const int64_t* L2 = lims + s2 * (nq + 1);
        if (s2 != s) slot += range_merge_rank(D + b2 + L2[q], L2[q + 1] - L2[q], v, maximize != 0, s2 < s);
        b2 += L2[nq];
    }
    outD[slot] = v;
    outP[slot] = P[i];
    order[slot] = i;
}

void dfx_range_merge_impl(int64_t S, int64_t nq, const int64_t* d_lims, const float* d_D, const int64_t* d_P,
                          int64_t total, int maximize, int64_t* d_out_lims, float* d_outD, int64_t* d_outP,
                          int64_t* d_order, cudaStream_t st) {
    DFX_REQUIRE(S >= 1 && nq >= 0 && total >= 0, "range merge: bad S / nq / total");
    DFX_REQUIRE(total <= (((int64_t)1 << 31) - 1) * 256, "range merge: too many entries");  // gridDim.x <= 2^31 - 1
    DFX_LAUNCH(range_merge_lims_kernel, 1, 256, 0, st, S, nq, d_lims, d_out_lims);
    if (total == 0 || nq == 0) return;
    DFX_LAUNCH(range_merge_kernel, (unsigned)dfx_ceil_div(total, 256), 256, 0, st, S, nq, total, d_lims, d_D, d_P,
               maximize, d_out_lims, d_outD, d_outP, d_order);
}

// =====================================================================================
// K7a: fused nearest-centroid assignment (build path).  Same FFMA tile as K1a, but the
// epilogue reduces each row's tile to one composite (value, column) and folds it into
// best[row] with a 64-bit atomicMin -- the values matrix is never written.  The minimum of
// composites is exactly the oracle's argmin with ties -> smaller index.
// =====================================================================================
template <int BM, int BN, int BK, int TM, int TN>
__global__ void __launch_bounds__((BM / TM) * (BN / TN))
gemm_argmin_kernel(const float* __restrict__ Q, int64_t nq, const float* __restrict__ X,
                   const float* __restrict__ xnorm, int64_t ncols, int d, int metric,
                   unsigned long long* __restrict__ best) {
    const int tid = threadIdx.x;
    const int tx = tid % (BN / TN), ty = tid / (BN / TN);
    const int64_t m0 = (int64_t)blockIdx.y * BM;
    const int64_t n0 = (int64_t)blockIdx.x * BN;
    float acc[TM][TN];
    gemm_tile_ffma<BM, BN, BK, TM, TN>(Q, nq, X, ncols, d, m0, n0, tx, ty, acc);
    constexpr int TXN = BN / TN;  // threads sharing a row (consecutive lanes)
#pragma unroll
    for (int i = 0; i < TM; i++) {
        unsigned long long c = DFX_COMP_NONE;
#pragma unroll
        for (int j = 0; j < TN; j++) {
            int64_t gn = n0 + tx * TN + j;
            if (gn < ncols) {
                unsigned long long cc = dfx_comp(dfx_rank_value(acc[i][j], metric, xnorm, gn), (uint32_t)gn);
                c = cc < c ? cc : c;
            }
        }
#pragma unroll
        for (int off = TXN / 2; off >= 1; off >>= 1) {
            unsigned long long o = __shfl_xor_sync(0xffffffffu, c, off);
            c = o < c ? o : c;
        }
        int64_t gm = m0 + ty * TM + i;
        if (tx == 0 && gm < nq && c != DFX_COMP_NONE) atomicMin(&best[gm], c);
    }
}

__global__ void unpack_best_kernel(const unsigned long long* __restrict__ best, int64_t n,
                                   int32_t* __restrict__ out) {
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) out[i] = (int32_t)(uint32_t)best[i];
}

void dfx_launch_assign_fused(const float* X, int64_t n, const float* cent, const float* cnorm,
                             int64_t nlist, int d, int metric, unsigned long long* best,
                             int32_t* out, cudaStream_t st) {
    if (n <= 0) return;
    DFX_CUDA(cudaMemsetAsync(best, 0xff, (size_t)n * 8, st));
    constexpr int BM = 128, BN = 128, BK = 8, TM = 8, TN = 8;
    static_assert(BN / TN == 16, "row group must be 16 consecutive lanes");
    const int64_t max_y = 65535;
    for (int64_t r0 = 0; r0 < n; r0 += max_y * BM) {
        int64_t rc = std::min<int64_t>(n - r0, max_y * BM);
        dim3 grid((unsigned)dfx_ceil_div(nlist, BN), (unsigned)dfx_ceil_div(rc, BM));
        auto kern = gemm_argmin_kernel<BM, BN, BK, TM, TN>;
        DFX_LAUNCH(kern, grid, (BM / TM) * (BN / TN), 0, st, X + r0 * d, rc, cent, cnorm, nlist, d, metric,
                   best + r0);
    }
    DFX_LAUNCH(unpack_best_kernel, (unsigned)dfx_ceil_div(n, 256), 256, 0, st, best, n, out);
}
