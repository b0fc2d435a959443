// dfx_tc.cu -- K1: the coarse quantizer on Hopper tensor cores (wgmma + TMA + mbarrier).
//
// Replaces the dense query x centroid contraction inside `quantizer.search(nq, x, nprobe)`
// (faiss IndexIVF::search, reached from reference distributed_faiss/index.py:257) and
// `quantizer.assign` (IndexIVF::add, index.py:425).
//
// Scheme ("screen on tensor cores, decide in canonical fp32"):
//   1. both operands are scaled by a power of two (queries per row, the table as a whole, so that
//      every row norm lands in [2^13, 2^14)) and rounded to fp16; q.c is accumulated in fp32
//      registers by wgmma: PRECISE splits each operand into fp16 hi + lo planes (three MMAs per
//      k-step), FAST uses the hi planes alone (one MMA).  The rounding error is bounded rigorously
//      for both, see screen_tol_rel.  The decide stage makes the result exact for ANY bounded
//      error; AUTO (the default) starts PRECISE and moves to FAST where FAST rarely overflows.
//   2. the epilogue turns each 128x128 accumulator tile into ranking values
//      (L2: |c|^2 - 2 q.c, IP: -q.c) and keeps only the MINIMUM of every group of 32
//      consecutive centroids -> gmin[nq][nlist/32]  (32x less traffic than the full matrix).
//   3. the G = nprobe + margin groups with the smallest minima are selected exactly
//      (dfx_select.cuh).  Every true top-nprobe centroid lies in a group whose minimum is within
//      the tolerance of the nprobe-th smallest minimum; if the G-th selected group is still within
//      it (more than `margin` near-ties, e.g. duplicate centroids) the row is re-done exactly by
//      tc_exact_rows_kernel -- nothing is ever dropped silently.
//   4. the candidate centroids are re-evaluated in the CANONICAL fp32 order
//      (seq-k FMA, identical to oracle/dfx_oracle.c) and the final top-nprobe / argmin is
//      taken on those exact values -> the probe lists are bit-identical to the oracle's.
//
// One CTA = 9 warps: warps 0..7 are two consumer warpgroups (warpgroup w owns query rows
// 64w..64w+63 of the 128-row tile: m64n128k16 wgmma into 64 fp32 registers per thread, then the
// epilogue on those registers), warp 8 is the TMA producer.  d <= 256: A (the query tile) stays
// resident in shared memory and B (centroids) streams through a ring of 16 KB stages; larger d
// (config C4, d = 768): A and B k-atoms stream through the ring together.
#include "dfx_internal.h"
#include <cmath>
#include <utility>
#include "dfx_select.cuh"
#include "dfx_topk.cuh"
#include "dfx_ptx.cuh"
#ifndef DFX_EMU
#include <cuda.h>
#endif

#ifndef DFX_EMU  // wgmma / TMA / mbarrier PTX: hardware only (the CPU emulator uses emu_tc_screen below)
// ------------------------------------------------------------------ PTX wrappers
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
    return (uint32_t)__cvta_generic_to_shared(p);
}
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
                 : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    const uint32_t addr = smem_u32(bar);
    uint32_t done;
    do {
        asm volatile(
            "{\n\t.reg .pred p;\n\t"
            "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
            "selp.u32 %0, 1, 0, p;\n\t}"
            : "=r"(done)
            : "r"(addr), "r"(parity)
            : "memory");
    } while (!done);
}
__device__ __forceinline__ void tma_load_2d(void* smem_dst, const CUtensorMap* tm, uint64_t* bar, int c0,
                                            int c1) {
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
        ::"r"(smem_u32(smem_dst)), "l"((uint64_t)tm), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
        : "memory");
}
__device__ __forceinline__ void wg_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
// wait until at most N committed wgmma groups of this warpgroup are still in flight
template <int N>
__device__ __forceinline__ void wg_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// D[64 x 128] (+)= A[64 x 16] . B[128 x 16]^T, fp16 operands from shared memory (both K-major),
// fp32 accumulator in registers (the m64nNk16 fragment layout: d[4j + 2h + e] holds row
// 16 warp + lane/4 + 8h, column 8j + 2 (lane & 3) + e)
__device__ __forceinline__ void wgmma_f16_n128(float (&d)[64], uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "setp.ne.b32 p, %66, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1, 0, 0;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
          "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
          "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
          "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
          "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
          "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
          "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
          "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
        : "l"(adesc), "l"(bdesc), "r"(accumulate)
        : "memory");
}
// The two smallest of a pair of packed ranking values merged into (m1, m2):
// m2 = min(m2, max(m1, lo), hi), m1 = min(m1, lo)
__device__ __forceinline__ void tc_pair_step(float a, float b, float& m1, float& m2) {
    const float lo = fminf(a, b), hi = fmaxf(a, b);
    m2 = fminf(fminf(m2, fmaxf(m1, lo)), hi);
    m1 = fminf(m1, lo);
}
// (bits(v) & mask) | idx in one LOP3 (mask in a register)
__device__ __forceinline__ float tc_pack_col(float v, uint32_t mask, uint32_t idx) {
    uint32_t r;
    asm("lop3.b32 %0, %1, %2, %3, 0xEA;" : "=r"(r) : "r"(__float_as_uint(v)), "r"(mask), "r"(idx));
    return __uint_as_float(r);
}
// (bits(v) & mask) | (bits(old) & ~mask) in one LOP3: v with the column bits of old
__device__ __forceinline__ float tc_repack(float v, uint32_t mask, float old) {
    uint32_t r;
    asm("lop3.b32 %0, %1, %2, %3, 0xE2;" : "=r"(r) : "r"(__float_as_uint(v)), "r"(mask), "r"(__float_as_uint(old)));
    return __uint_as_float(r);
}

// K-major, SWIZZLE_128B shared-memory matrix descriptor (rows of 128 B, 8-row atoms of 1024 B)
__device__ __forceinline__ uint64_t make_kmajor_sw128_desc(uint32_t smem_addr) {
    uint64_t d = 0;
    d |= (uint64_t)((smem_addr & 0x3ffffu) >> 4);  // start address, 16-byte units
    d |= (uint64_t)1 << 16;                        // leading byte offset (unused with a 128-byte swizzle)
    d |= (uint64_t)(1024u >> 4) << 32;             // stride byte offset between 8-row atoms
    d |= (uint64_t)1 << 62;                        // SWIZZLE_128B
    return d;
}

#endif  // !DFX_EMU

// ------------------------------------------------------------------ the kernel
namespace tc {
constexpr int TILE = 128;           // rows of A and of B per tile
constexpr int KATOM = 64;           // fp16 elements per 128-byte swizzle row
constexpr int ATOM_BYTES = TILE * KATOM * 2;  // 16 KB
constexpr int CONSUMERS = 256;      // two warpgroups, 64 query rows each
constexpr int THREADS = CONSUMERS + 32;  // + the TMA producer warp
constexpr int MAX_RESIDENT_KATOMS = 4;  // query tile resident in shared memory up to 4 atoms (64 KB): FAST d <= 256, PRECISE d <= 128
// Screening precision (NPL = planes per operand):
//   FAST    NPL 1: fp16(x s); one MMA per k-step; error <= |q||c| (2^-10 + 2^-13)
//   PRECISE NPL 2: hi = fp16(x s), lo = fp16(x s - hi); q.c ~= qh.ch + ql.ch + qh.cl, three MMAs per
//           k-step; error <= |q||c| 2^-17 (the dropped ql.cl term is 2^-22, hi + lo carries 22 bits)
// shared-memory plan (offsets inside the 1024-aligned dynamic block)
//   resident A (NPL x katoms <= 4): A = NPL x katoms x 16 KB, then a ring of B stages of 16 KB that
//                          holds two tiles, at least 4 stages (FAST d <= 128: <= 103 KB, two CTAs per
//                          SM; PRECISE d = 128 and FAST d = 256: 8 stages, 199 KB); the warpgroups run
//                          a tile apart, and the one behind still reads the stages of the tile before
//   streamed A (larger d): a ring of 6 stages of (A atom + B atom) = 32 KB
//   then 512 B of mbarriers, each warpgroup's copy of the tile's ranking offsets, [2][2][TILE] floats,
//   and the held summary of an even tile, [CONSUMERS / 2][2] float4 (4 KB)
struct Smem {
    static constexpr bool resident(int katoms, int npl) { return npl * katoms <= MAX_RESIDENT_KATOMS; }
    static constexpr int nstage(bool res, int katoms, int npl) {
        return !res ? 6 : (2 * npl * katoms > 4 ? 2 * npl * katoms : 4);
    }
    static constexpr int stage_bytes(bool res) { return res ? ATOM_BYTES : 2 * ATOM_BYTES; }
    static constexpr int RING(bool res, int katoms, int npl) { return res ? npl * katoms * ATOM_BYTES : 0; }
    static constexpr int BARS(bool res, int katoms, int npl) { return RING(res, katoms, npl) + nstage(res, katoms, npl) * stage_bytes(res); }
    static constexpr int HELD(bool res, int katoms, int npl) { return BARS(res, katoms, npl) + 512 + 4 * TILE * 4; }
    static constexpr int total(bool res, int katoms, int npl) { return HELD(res, katoms, npl) + CONSUMERS / 2 * 32; }
    // CTAs that fit one SM (228 KB of shared memory): two when a CTA's block (+ 1 KB for the
    // alignment) stays within 113 KB, which only FAST shapes reach
    static constexpr int ctas_per_sm(bool res, int katoms, int npl) {
        return (npl == 1 && total(res, katoms, npl) + 1024 <= 113 * 1024) ? 2 : 1;
    }
};
}  // namespace tc

// the power of two that brings a norm into [2^13, 2^14) (1 for a zero / non-finite norm; the
// exponent is clamped to +-45, norms beyond 2^+-45 are outside what the screening supports)
__host__ __device__ __forceinline__ float dfx_pow2_scale(float nrm) {
    if (!(nrm > 0.f) || !(nrm < 3.0e38f)) return 1.f;
    int e;
    frexpf(nrm, &e);  // nrm = m 2^e, m in [0.5, 1)
    e = e < -45 ? -45 : (e > 45 ? 45 : e);
    return ldexpf(1.f, 14 - e);
}

__device__ __forceinline__ double tc_warp_sum(double v) {
#pragma unroll
    for (int off = 16; off >= 1; off >>= 1) v += __shfl_xor_sync(0xffffffffu, v, off);
    return v;
}

// Centring.  |c|^2 - 2 q.c = -2 (q-m).(c-m) + |c-m|^2 + (|m|^2 - 2 q.m) and
// -q.c = -(q-m).(c-m) - m.c + (|m|^2 - q.m) hold for any m: the tensor cores take the centred
// operands, the epilogue adds a column term (|c-m|^2 or -m.c) and a row term.  The screening
// error scales with |q-m| max|c-m| instead of |q| max|c|, far smaller where the rows share a
// large common mean.  m = the mean of the table's rows, summed in fp64 (deterministically: row
// slices, then the slices in order).
constexpr int MEAN_CHUNKS = 128;
__global__ void __launch_bounds__(256)
col_part_kernel(const float* __restrict__ x, int64_t n, int d, double* __restrict__ part) {
    __shared__ double s[8][32];
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    const int k = blockIdx.x * 32 + lane;  // d % 32 == 0
    const int64_t per = (n + MEAN_CHUNKS - 1) / MEAN_CHUNKS;
    const int64_t r0 = (int64_t)blockIdx.y * per, r1 = r0 + per < n ? r0 + per : n;
    double acc = 0.0;
    for (int64_t r = r0 + w; r < r1; r += 8) acc += (double)x[r * d + k];
    s[w][lane] = acc;
    __syncthreads();
    if (w == 0) {
        double t = 0.0;
        for (int i = 0; i < 8; i++) t += s[i][lane];
        part[(int64_t)blockIdx.y * d + k] = t;
    }
}
__global__ void col_mean_kernel(const double* __restrict__ part, int d, int64_t n, float* __restrict__ mean) {
    const int k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= d) return;
    double t = 0.0;
    for (int c = 0; c < MEAN_CHUNKS; c++) t += part[(int64_t)c * d + k];
    mean[k] = n > 0 ? (float)(t / (double)n) : 0.f;
}
// per table row (one warp per row, fp64 sums rounded once): the column term, L2 |x-m|^2 or IP
// -m.x (3e38 for the padded rows: never selected), and maxima[0..1] = max |x|^2, max |x-m|^2
// (atomicMax on the bits of non-negative floats)
__global__ void __launch_bounds__(256)
table_terms_kernel(const float* __restrict__ x, int64_t n, int64_t n_pad, int d, const float* __restrict__ mean,
                   int metric, float* __restrict__ cterm, float* __restrict__ maxima) {
    const int lane = threadIdx.x & 31;
    const int64_t row = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (row >= n_pad) return;
    if (row >= n) {
        if (lane == 0) cterm[row] = 3.0e38f;
        return;
    }
    double n2 = 0.0, n2c = 0.0, xm = 0.0;
    for (int k = lane; k < d; k += 32) {
        const double v = x[row * d + k], mk = mean[k];
        n2 += v * v;
        n2c += (v - mk) * (v - mk);
        xm += v * mk;
    }
    n2 = tc_warp_sum(n2);
    n2c = tc_warp_sum(n2c);
    xm = tc_warp_sum(xm);
    if (lane == 0) {
        cterm[row] = metric == DFX_METRIC_L2 ? (float)n2c : (float)(-xm);
        atomicMax(reinterpret_cast<int*>(maxima), __float_as_int((float)n2));
        atomicMax(reinterpret_cast<int*>(maxima) + 1, __float_as_int((float)n2c));
    }
}

// fp32 rows minus m -> fp16 rows scaled by a power of two, rows >= n zero filled; one warp per row.
//   row_scaled != 0 (queries): the row is scaled so that its centred norm lands in [2^13, 2^14);
//       mult[row] = factor / (row scale * table_scale) is what the screening epilogue multiplies
//       the accumulator with (factor = -2 for L2, -1 for inner product; all powers of two, exact),
//       qterm[row] = |m|^2 + factor q.m the row term it adds, qn[row] = (|q|^2, |q-m|^2) for the
//       tolerance (fp64 sums, rounded once; zero for padded rows);
//   row_scaled == 0 (a screening table): every row times table_scale.
// x - m is rounded to fp32 before the scaling (a power of two, exact).  Elements more than 2^28
// below the row norm fall into fp16's subnormal range and lose relative (not absolute)
// precision: an error of at most 2^-39 of the norm, far inside screen_tol.
// npl == 2 also writes the residual plane lo = fp16(v - hi) at out + n_pad * d.
__global__ void __launch_bounds__(256)
f16_rows_kernel(const float* __restrict__ x, int64_t n, int64_t n_pad, int d, const float* __restrict__ mean,
                int row_scaled, float table_scale, float factor, int npl, __half* __restrict__ out,
                float* __restrict__ mult, float2* __restrict__ qn, float* __restrict__ qterm) {
    const int lane = threadIdx.x & 31;
    const int64_t row = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (row >= n_pad) return;
    const bool real = row < n;
    float scale = table_scale;
    if (row_scaled) {
        double n2 = 0.0, n2c = 0.0, qm = 0.0, mm = 0.0;
        if (real)
            for (int k = lane; k < d; k += 32) {
                const double v = x[row * d + k], mk = mean[k];
                n2 += v * v;
                n2c += (v - mk) * (v - mk);
                qm += v * mk;
                mm += mk * mk;
            }
        n2 = tc_warp_sum(n2);
        n2c = tc_warp_sum(n2c);
        qm = tc_warp_sum(qm);
        mm = tc_warp_sum(mm);
        scale = dfx_pow2_scale(sqrtf((float)n2c));
        if (lane == 0) {
            mult[row] = factor / (scale * table_scale);
            qn[row] = make_float2((float)n2, (float)n2c);
            qterm[row] = (float)(mm + (double)factor * qm);
        }
    }
    for (int k = lane; k < d; k += 32) {
        const float v = real ? (x[row * d + k] - mean[k]) * scale : 0.f;
        const __half hi = __float2half_rn(v);
        out[row * d + k] = hi;
        if (npl == 2) out[n_pad * d + row * d + k] = __float2half_rn(v - __half2float(hi));
    }
}

#ifdef DFX_EMU
// ---- CPU emulator stand-in (tests/emu/): the screening kernel cannot be emulated instruction
// by instruction, so its RESULT is restated: the centred fp16 operands the product code prepared
// (f16_rows_kernel), fp32 accumulation (order not specified by the hardware either), the
// epilogue's centred ranking value fma(acc, mult[row], cterm[col]), its packed (min, runner-up,
// arg-min) per 32 centroids, and the row term added to the minimum and runner-up with their
// column bits kept.  Everything downstream (group selection, exact canonical re-evaluation, the
// overflow fallback, the drivers) is the product code.  one: the table is one exact plane of ncols rows
// (the kernel's ONE: PRECISE accumulates qh.c + ql.c); the column term as the kernel reads it.
static void emu_tc_screen(const __half* qh, const float* qmult, const float* qterm, int64_t nq, int64_t nq_pad,
                          const __half* ch, int64_t nl_pad, int64_t ncols, bool one, int d, int npl,
                          const float* cterm, float* gmin, float* gmin2, uint8_t* gargc, float* tmin, int ng) {
    const float big = 3.0e38f;
    auto repack = [](float v, float col_of) {  // v with the 5 low bits of col_of
        uint32_t u, c;
        memcpy(&u, &v, 4);
        memcpy(&c, &col_of, 4);
        u = (u & ~31u) | (c & 31u);
        memcpy(&v, &u, 4);
        return v;
    };
    std::vector<float> cf((size_t)npl * nl_pad * d, 0.f), qf((size_t)npl * d);
    const size_t present = one ? (size_t)ncols * d : cf.size();  // one plane: rows >= ncols read as zeros
    for (size_t i = 0; i < present; i++) cf[i] = __half2float(ch[i]);
    for (int64_t row = 0; row < nq; row++) {
        for (int pl = 0; pl < npl; pl++)
            for (int k = 0; k < d; k++) qf[(size_t)pl * d + k] = __half2float(qh[(size_t)pl * nq_pad * d + row * d + k]);
        for (int g = 0; g < ng; g++) {
            float m1 = big, m2 = big;
            for (int j = 0; j < 32; j++) {
                const int64_t col = (int64_t)g * 32 + j;
                float acc = 0.f;
                const float* h = &cf[(size_t)col * d];
                for (int k = 0; k < d; k++) acc += qf[k] * h[k];
                if (npl == 2) {
                    const float* l = &cf[(size_t)nl_pad * d + (size_t)col * d];
                    for (int k = 0; k < d; k++) acc += qf[d + k] * h[k] + (one ? 0.f : qf[k] * l[k]);
                }
                const float ct = col < ncols ? (cterm ? cterm[col] : 0.f) : big;
                const float v = fmaf(acc, qmult[row], ct);
                uint32_t u;
                memcpy(&u, &v, 4);
                u = (u & ~31u) | (uint32_t)j;
                float vj;
                memcpy(&vj, &u, 4);
                m2 = fminf(m2, fmaxf(m1, vj));
                m1 = fminf(m1, vj);
            }
            m1 = repack(m1 + qterm[row], m1);
            m2 = repack(m2 + qterm[row], m2);
            uint32_t u1;
            memcpy(&u1, &m1, 4);
            gmin[row * ng + g] = m1;
            gmin2[row * ng + g] = m2;
            gargc[row * ng + g] = (uint8_t)(u1 & 31u);
        }
        for (int t = 0; t < ng / 4; t++) {  // the minimum of every tile of 4 groups
            const float* gm = gmin + row * ng + 4 * t;
            tmin[row * (ng / 4) + t] = fminf(fminf(gm[0], gm[1]), fminf(gm[2], gm[3]));
        }
    }
}
#else
// tmQ: fp16 [NPL * nq_pad, d] (scaled query rows; NPL == 2: hi plane then lo plane), tmC: fp16
// [NPL * nl_pad, d] (scaled table rows), d = 64 KATOMS
// qmult, qterm: float [nq_pad], the per-row multiplier of the accumulator and the row term
// (f16_rows_kernel); cterm: float [nl_pad], the column term (padded with 3e38)
// gmin / gmin2: float [nq][ng], gargc: u8 [nq][ng], ng = nl_pad/32
// KT: d / 64 at compile time for the resident shapes (1, 2, 4); 0 = streamed, k-atoms at run time
// ONE: the table is one exact fp16 plane (FLAT_SQ16 rows, tmC [ncols, d]) -- PRECISE is then (qh, c) and
// (ql, c), two MMAs per k-step; FAST (NPL 1) is the same kernel for either table
// cterm: column c < ncols reads cterm[c] (0 when cterm is null), columns >= ncols are never selected
template <int KT, int NPL, bool ONE = false>
__global__ void __launch_bounds__(tc::THREADS, KT != 0 ? tc::Smem::ctas_per_sm(true, KT, NPL) : 1)
tc_coarse_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmC, int nq,
                 int nq_pad, int nl_pad, int ncols, int katoms_rt, const float* __restrict__ cterm,
                 const float* __restrict__ qmult, const float* __restrict__ qterm, int ctiles_per_cta,
                 float* __restrict__ gmin, float* __restrict__ gmin2, uint8_t* __restrict__ gargc,
                 float* __restrict__ tmin, int ng) {
    using namespace tc;
    constexpr bool RES = KT != 0;
    const int KATOMS = KT ? KT : katoms_rt;
    constexpr int NSTAGE = Smem::nstage(RES, KT, NPL);
    constexpr int STAGE_BYTES = Smem::stage_bytes(RES);
    constexpr int TN = TILE;  // centroids per tile
    // operand pairs accumulated per k-atom: FAST (qh, ch); PRECISE (qh, ch), (ql, ch), (qh, cl) -- or,
    // with an exact table plane, (qh, c), (ql, c)
    constexpr int NCOMBO = NPL == 1 ? 1 : ONE ? 2 : 3;
    constexpr int NBPL = ONE ? 1 : NPL;  // table planes
    extern __shared__ unsigned char smem_raw_tc[];
    unsigned char* smem = reinterpret_cast<unsigned char*>(
        (reinterpret_cast<uintptr_t>(smem_raw_tc) + 1023) & ~(uintptr_t)1023);  // SWIZZLE_128B atoms
    unsigned char* sA = smem;                            // RES: [plane][katom] x 16 KB
    unsigned char* sR = smem + Smem::RING(RES, KATOMS, NPL);  // ring: B atom (RES) or A atom + B atom
    uint64_t* bars = reinterpret_cast<uint64_t*>(smem + Smem::BARS(RES, KATOMS, NPL));
    uint64_t* full = bars;                 // [NSTAGE]
    uint64_t* empty = bars + NSTAGE;       // [NSTAGE]
    uint64_t* a_full = bars + 2 * NSTAGE;  // [1]
    float* s_cn = reinterpret_cast<float*>(smem + Smem::BARS(RES, KATOMS, NPL) + 512);  // [warpgroup][2][TN]
    float4* s_held = reinterpret_cast<float4*>(smem + Smem::HELD(RES, KATOMS, NPL));   // [CONSUMERS / 2][2]

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int qt = blockIdx.y;
    const int ctiles = nl_pad / TN;
    const int ct0 = blockIdx.x * ctiles_per_cta;
    const int ct1 = min(ctiles, ct0 + ctiles_per_cta);
    const int ntiles = ct1 - ct0;
    if (ntiles <= 0) return;

    if (threadIdx.x == 0) {
        for (int i = 0; i < NSTAGE; i++) {
            mbar_init(&full[i], 1);
            mbar_init(&empty[i], CONSUMERS / 32);  // one arrival per consumer warp
        }
        mbar_init(a_full, 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    }
    __syncthreads();

    if (warp == CONSUMERS / 32) {
        // ===================== TMA producer =====================
        // RES: per tile, the B atoms of the hi plane then (PRECISE, two table planes) of the lo plane.
        // streamed: per tile and k-atom, the (A atom, B atom) pair of every combo.
        if (lane == 0) {
            if (RES) {
                mbar_expect_tx(a_full, NPL * KATOMS * ATOM_BYTES);
                for (int pl = 0; pl < NPL; pl++)
                    for (int ka = 0; ka < KATOMS; ka++)
                        tma_load_2d(sA + (pl * KATOMS + ka) * ATOM_BYTES, &tmQ, a_full, ka * KATOM,
                                    pl * nq_pad + qt * TILE);
            }
            int stage = 0, phase = 0;
            for (int t = 0; t < ntiles; t++) {
                const int crow = (ct0 + t) * TN;
                // RES: c = B plane; streamed: c = combo
                for (int c = 0; c < (RES ? NBPL : NCOMBO); c++)
                for (int ka = 0; ka < KATOMS; ka++) {
                    mbar_wait(&empty[stage], phase ^ 1);
                    mbar_expect_tx(&full[stage], STAGE_BYTES);
                    unsigned char* dst = sR + stage * STAGE_BYTES;
                    if (!RES) {
                        tma_load_2d(dst, &tmQ, &full[stage], ka * KATOM, (c == 1 ? nq_pad : 0) + qt * TILE);
                        dst += ATOM_BYTES;
                    }
                    const int bpl = RES ? c : (c == 2 ? 1 : 0);
                    tma_load_2d(dst, &tmC, &full[stage], ka * KATOM, bpl * nl_pad + crow);
                    if (++stage == NSTAGE) {
                        stage = 0;
                        phase ^= 1;
                    }
                }
            }
        }
        return;
    }

    // ===================== consumers: MMA, then registers -> per-group (min, runner-up, argmin) ====
    // The column index (0..31) inside its group replaces the 5 low mantissa bits of the screening
    // value (a 2^-18 relative perturbation, inside the screening tolerance), which makes the
    // arg-min fall out of the minimum itself.
    const int wg = warp >> 2;                  // warpgroup: query rows 64 wg .. 64 wg + 63
    const int quad = lane & 3;                 // the 4 lanes of a quad share a row
    const int row0 = wg * 64 + (warp & 3) * 16 + (lane >> 2);  // rows row0 and row0 + 8 of the tile
    const int64_t grow0 = (int64_t)qt * TILE + row0;
    const float big = 3.0e38f;                 // out-of-range columns: finite, never selected
    const float mult0 = qmult[grow0], mult1 = qmult[grow0 + 8];  // padded rows carry a multiplier too
    const float rq0 = qterm[grow0], rq1 = qterm[grow0 + 8];
    uint32_t idx_mask;                         // ~31 in a REGISTER: (v & mask) | j is then one LOP3
    asm volatile("mov.u32 %0, 0xffffffe0;" : "=r"(idx_mask));
    const uint32_t a_off = (uint32_t)wg * (TILE / 2) * 128;  // this warpgroup's 64 rows of an A atom
    const uint32_t a_base = smem_u32(sA) + a_off;
    const uint32_t r_base = smem_u32(sR);
    if (RES) mbar_wait(a_full, 0);
    int stage = 0, phase = 0;
    float acc[64];
    // The summary of an even centroid tile is held until the odd tile after it is done: lane q of
    // a quad then writes row row0 + 8 (q >> 1) of tile parity q & 1, so that adjacent lanes fill one
    // sector of each array in one store.  The stores, not the arithmetic, bounded the epilogue:
    // one partial sector per array, row and tile.  Lanes of parity 0 hold (gmin, gmin2) of their
    // row in shared memory (registers would spill under the two-CTA cap).
    const int hq = quad >> 1, pq = quad & 1;
    const int64_t grow_q = grow0 + 8 * hq;
    float4* held = s_held + 2 * (threadIdx.x >> 1);  // parity-0 lanes: [gmin, gmin2]
    // one wgmma group stays in flight while the next stage is awaited: a stage is released once
    // the group after it has been issued and the group that read it has completed
    auto release = [&](int s) {
        __syncwarp();
        if (lane == 0) mbar_arrive(&empty[s]);  // this warp's MMAs have read stage s
    };
    // Resident shapes: the two warpgroups run out of phase -- while one turns its accumulator into
    // the summary, the other's MMAs keep the tensor cores busy.  The turn to issue a tile's MMAs
    // passes back and forth through named barriers 2 (warpgroup 0 waits, from its second tile on)
    // and 3 (warpgroup 1 waits), so the MMAs of the two never interleave.  The streamed ring holds
    // less than a tile: there both warpgroups issue together.
    for (int t = 0; t < ntiles; t++) {
        const int buf = t & 1;
        const int col0 = (ct0 + t) * TN;
        // the column term of column threadIdx.x % 128 of the tile (`big` past nlist); loaded now,
        // shared through this warpgroup's copy once the MMAs are issued
        const int own_col = col0 + (threadIdx.x & (TN - 1));
        const float cn_own = own_col < ncols ? (cterm ? cterm[own_col] : 0.f) : big;
        if (RES && (wg == 1 || t > 0)) asm volatile("bar.sync %0, %1;" ::"r"(2 + wg), "n"(CONSUMERS) : "memory");
        int prev = -1;  // stage of the group still in flight
        for (int c = 0; c < (RES ? NBPL : NCOMBO); c++)
        for (int ka = 0; ka < KATOMS; ka++) {
            mbar_wait(&full[stage], phase);
            const uint32_t st_addr = r_base + stage * STAGE_BYTES;
            const uint32_t b_addr = RES ? st_addr : st_addr + ATOM_BYTES;
            const uint32_t ah_addr = RES ? a_base + ka * ATOM_BYTES : st_addr + a_off;
            const uint32_t al_addr = a_base + (KATOMS + ka) * ATOM_BYTES;  // RES && NPL == 2 only
            wg_fence();
#pragma unroll
            for (int kk = 0; kk < KATOM / 16; kk++) {  // k16 per wgmma = 32 bytes of a swizzle row
                const uint64_t bd = make_kmajor_sw128_desc(b_addr + kk * 32);
                wgmma_f16_n128(acc, make_kmajor_sw128_desc(ah_addr + kk * 32), bd,
                               (c > 0 || ka > 0 || kk > 0) ? 1u : 0u);
                // resident PRECISE: the hi-plane B stage also takes ql . ch
                if (RES && NPL == 2 && c == 0) wgmma_f16_n128(acc, make_kmajor_sw128_desc(al_addr + kk * 32), bd, 1u);
            }
            wg_commit();
            wg_wait<1>();  // the group issued before this one has completed
            if (prev >= 0) release(prev);
            prev = stage;
            if (++stage == NSTAGE) {
                stage = 0;
                phase ^= 1;
            }
        }
        if (RES && (wg == 0 || t + 1 < ntiles))
            asm volatile("bar.arrive %0, %1;" ::"r"(3 - wg), "n"(CONSUMERS) : "memory");
        float* cn_wg = s_cn + (wg * 2 + buf) * TN;
        cn_wg[threadIdx.x & (TN - 1)] = cn_own;
        wg_wait<0>();  // the accumulator is complete
        release(prev);
        // this warpgroup's offsets written (its copy of tile t - 2 was read before tile t - 1's barrier)
        asm volatile("bar.sync %0, %1;" ::"r"(4 + wg), "n"(CONSUMERS / 2) : "memory");
        const float* cn = cn_wg + 2 * quad;
        float gm[2][4], gm2[2][4];
        uint32_t ga[2] = {0u, 0u};
#pragma unroll
        for (int g = 0; g < 4; g++) {  // groups of 32 columns: fragments j = 4g .. 4g + 3
#pragma unroll
            for (int h = 0; h < 2; h++) {
                const float mult = h ? mult1 : mult0;
                float m1 = big, m2 = big;
#pragma unroll
                for (int jj = 0; jj < 4; jj++) {
                    const int j = 4 * g + jj;
                    const float2 c2 = *reinterpret_cast<const float2*>(cn + 8 * j);
                    const uint32_t ci = (uint32_t)(8 * jj + 2 * quad);
                    const float a = tc_pack_col(fmaf(acc[4 * j + 2 * h], mult, c2.x), idx_mask, ci);
                    const float b = tc_pack_col(fmaf(acc[4 * j + 2 * h + 1], mult, c2.y), idx_mask, ci + 1);
                    tc_pair_step(a, b, m1, m2);
                }
#pragma unroll
                for (int off = 1; off <= 2; off <<= 1) {  // the quad's four partial results
                    const float o1 = __shfl_xor_sync(0xffffffffu, m1, off);
                    const float o2 = __shfl_xor_sync(0xffffffffu, m2, off);
                    m2 = fminf(fmaxf(m1, o1), fminf(m2, o2));
                    m1 = fminf(m1, o1);
                }
                // back to the original ranking frame: + the row term, column bits kept
                const float rq = h ? rq1 : rq0;
                m1 = tc_repack(m1 + rq, idx_mask, m1);
                m2 = tc_repack(m2 + rq, idx_mask, m2);
                gm[h][g] = m1;
                gm2[h][g] = m2;
                ga[h] |= (__float_as_uint(m1) & 31u) << (8 * g);
            }
        }
        // every lane of a quad holds both rows' results; lane q takes row row0 + 8 (q >> 1)
        const float4 m = hq ? make_float4(gm[1][0], gm[1][1], gm[1][2], gm[1][3])
                            : make_float4(gm[0][0], gm[0][1], gm[0][2], gm[0][3]);
        const float4 m2 = hq ? make_float4(gm2[1][0], gm2[1][1], gm2[1][2], gm2[1][3])
                             : make_float4(gm2[0][0], gm2[0][1], gm2[0][2], gm2[0][3]);
        const uint32_t a = hq ? ga[1] : ga[0];
        const int ct = ct0 + t;                           // global index of this centroid tile
        if (!(ct & 1) && t + 1 < ntiles) {                // even tile with its odd partner to come
            if (pq == 0) {
                held[0] = m;
                held[1] = m2;
            }
            continue;
        }
        const bool pair = (ct & 1) && t > 0;              // the held even tile goes out with this one
        if ((pair || pq == 0) && grow_q < nq) {
            const bool old = pair && pq == 0;             // lane writes the held tile ct - 1
            const float4 wm = old ? held[0] : m, wm2 = old ? held[1] : m2;
            const int wct = old ? ct - 1 : ct;
            const int64_t o = grow_q * ng + 4 * wct;
            *reinterpret_cast<float4*>(gmin + o) = wm;
            *reinterpret_cast<float4*>(gmin2 + o) = wm2;
            // gmin carries its arg-min column in its 5 low bits
            *reinterpret_cast<uint32_t*>(gargc + o) =
                old ? (__float_as_uint(wm.x) & 31u) | (__float_as_uint(wm.y) & 31u) << 8 |
                          (__float_as_uint(wm.z) & 31u) << 16 | (__float_as_uint(wm.w) & 31u) << 24
                    : a;
            // the tile's minimum: the first level of the group selection (topg_collect_kernel)
            tmin[grow_q * (ng >> 2) + wct] = fminf(fminf(wm.x, wm.y), fminf(wm.z, wm.w));
        }
    }
}
#endif  // DFX_EMU

// Which columns of the selected groups can still matter?  With t = value of the nprobe-th
// smallest group minimum and tol >= twice the screening error, every true top-nprobe centroid c
// has approx(c) <= t + tol; inside its group it is either the arg-min column or has
// approx(c) >= gmin2(group).  So a group is expanded to all 32 columns only if
// gmin2 <= t + tol, otherwise its arg-min column is the only candidate.
//
// The tolerance must be twice the error e of one value against its canonical value (threshold
// and candidate are both approximations), up to a constant per row (it moves every value of the
// row alike).  With sc = |q-m| max|c-m|, Vc = max|c-m|^2 + 2 sc (bounds a centred value),
// s = |q| max|c| and V = max|c|^2 + 2 s (bounds a value in the original frame):
//   the centred product (q-m).(c-m) on the tensor cores, Cauchy-Schwarz bounding sum |q_k c_k|:
//     FAST (fp16 operands): every product carries two relative roundings of at most 2^-11
//       (2^-10 + 2^-22 together), the fp32 accumulation of the d products at most d 2^-24:
//         err = 2^-10 + 2^-22 + d 2^-24
//     PRECISE (hi + lo planes, three partial products): hi + lo represents an operand to 2^-22,
//       the dropped ql.cl term is 2^-22, 3d products are accumulated:
//         err = 3 2^-22 + 3 d 2^-24
//     plus 2^-23 for the fp32 subtractions q - m and c - m (2^-24 per operand); the L2 value
//     takes the product twice: 2 (err + 2^-23) sc;
//   in the centred frame, <= (2^-18 + 2^-23) Vc: the epilogue's fma (2^-24), the fp32 column
//     term (2^-24) and the packed column index (2^-18 of the value);
//   in the original frame, <= (2^-17 + 2^-22 + d 2^-24) V: the row term's addition (2^-24) and
//     the re-packed column index (2^-18); the canonical value's own rounding (d 2^-24 for |c|^2
//     and for q.c, 2^-24 for their difference), no longer shared with the screening value; for
//     inner product, where a centred value is bounded by V + Vc, the centred-frame terms on V.
// tol = 2 e, +5 % slack.  The row term itself (fp64, rounded once) is a constant per row.
//
// An exact table plane (FLAT_SQ16: the stored fp16 rows, m = 0, scale 1) drops the table's rounding
// and the subtractions: only the query is rounded, and q.c is accumulated from exact products:
//     FAST (qh . c, one MMA): err = 2^-11 + d 2^-24
//     PRECISE (qh . c + ql . c, two MMAs): qh + ql represents q to 2^-22, 2d products accumulated:
//         err = 2^-22 + 2 d 2^-24
// With m = 0 the centred and the original frame coincide (sc = s, Vc = V, the row term is 0), so the
// other two terms of screen_tol stand as they are; they still cover the epilogue's fma, the column
// term (for L2 the stored |x|^2, the very value the canonical one adds), the packed column index and
// the canonical value's own rounding.
static float screen_tol_rel(int d, bool fast, bool exact_table = false) {
    if (exact_table)
        return (float)(4.2 * (fast ? 1.0 / 2048 + d / 16777216.0 : 1.0 / 4194304 + 2.0 * d / 16777216.0));
    const double err = fast ? (1.0 / 1024 + 1.0 / 4194304 + d / 16777216.0) : (3.0 / 4194304 + 3.0 * d / 16777216.0);
    return (float)(4.2 * (err + 1.0 / 8388608));
}
static float screen_tol_raw(int d) { return (float)(2.1 * (1.0 / 131072 + 1.0 / 4194304 + d / 16777216.0)); }
constexpr float SCREEN_TOL_CENTRED = (float)(2.1 * (1.0 / 262144 + 1.0 / 8388608));
// what the tolerance of a row needs besides its precision: the table's maxima and the rows' norms
struct ScreenTol {
    float rel;            // of this launch's precision
    float rel_fast;       // > 0: also count the rows FAST would overflow
    float raw;            // screen_tol_raw(d)
    float cmax2, cmax2c;  // max |c|^2, max |c-m|^2
    const float2* qn;     // per row: |q|^2, |q-m|^2 (f16_rows_kernel)
};
__device__ __forceinline__ float screen_tol(const ScreenTol& t, int64_t row, float rel) {
    const float2 qn = t.qn[row];
    const float s = sqrtf(qn.x * t.cmax2), sc = sqrtf(qn.y * t.cmax2c);
    return rel * sc + SCREEN_TOL_CENTRED * (t.cmax2c + 2.f * sc) + t.raw * (t.cmax2 + 2.f * s) + 1e-30f;
}
// "the selected groups may not be all that matter": the G-th (last) selected group is itself
// within the tolerance, so an unselected group could be too -> the row is re-done exactly.
// last = the minimum of the G-th selected group, NaN (never within) when every group is selected.
__device__ __forceinline__ float screen_last_min(const int32_t* __restrict__ groups, int64_t row, int G, int ng,
                                                 const float* __restrict__ gmin) {
    const int gl = G < ng ? groups[row * G + G - 1] : -1;
    return gl >= 0 ? gmin[row * ng + gl] : __int_as_float(0x7fc00000);
}
// The decide threshold of a row, t + tol with t = the nprobe-th smallest group minimum (inf when
// there are fewer groups than probes: nothing is pruned).  A row with more near-ties than
// selected groups is queued for tc_exact_rows_kernel.  ovf = [overflow rows, rows that the FAST
// tolerance would overflow (counted by PRECISE launches for the AUTO mode), row list ...].
// t and last as the selection left them (decide_rows_kernel holds both in registers when it
// selects the groups itself).
__device__ __forceinline__ float screen_threshold(float t, float last, int64_t row, const ScreenTol& tol,
                                                  int32_t* __restrict__ ovf) {
    const float thr = t + screen_tol(tol, row, tol.rel);
    if (last <= thr) ovf[2 + atomicAdd(&ovf[0], 1)] = (int32_t)row;
    if (tol.rel_fast > 0.f && last <= t + screen_tol(tol, row, tol.rel_fast)) atomicAdd(&ovf[1], 1);
    return thr;
}
// the same from the selected groups in global memory ([rows][G], -1 = none)
__device__ __forceinline__ float screen_threshold(const int32_t* __restrict__ groups, int64_t row, int G, int nprobe,
                                                  int ng, const float* __restrict__ gmin, const ScreenTol& tol,
                                                  int32_t* __restrict__ ovf) {
    const int gk = (nprobe <= G) ? groups[row * G + nprobe - 1] : -1;
    const float t = gk >= 0 ? gmin[row * ng + gk] : __int_as_float(0x7f800000);
    return screen_threshold(t, screen_last_min(groups, row, G, ng, gmin), row, tol, ovf);
}
// Can a selected group (minimum m1, runner-up m2) still matter?  Only if its minimum is within
// the threshold (the return value); then through all 32 columns if its runner-up is within it
// too (expand, which means nothing for a group that is not live), otherwise through its arg-min
// column alone.
__device__ __forceinline__ bool group_live(float m1, float m2, float thr, bool& expand) {
    expand = m2 <= thr;
    return m1 <= thr;
}

// The G (<= 32) smallest group minima of a row, ascending by (value, group), by one warp: lane r
// gets the composite (value, group) of the r-th, NONE from lane G on.
//   1. every lane takes the minimum of its n/32 values; the G-th smallest of those 32 lane
//      minima, B, bounds the answer from above (G different lanes hold a value <= B);
//   2. the values <= B are collected (a few dozen at most in practice) into buf, the warp's CAP
//      slots of shared memory;
//   3. the buffer is bitonic-sorted by the warp and the first G entries are kept.
// Exact for any input; if more than CAP values are <= B (massive ties) the row falls back to
// G rounds of warp arg-min.  ~10x fewer instructions than G x n compare rounds.
// Two levels (fine != nullptr): `coarse` holds the minimum of every FINE_PER = 4 consecutive
// groups (one 128-column tile of the screening kernel, written by its epilogue) -- steps 1-3 run
// on the n / 4 tile minima, then the G smallest of the 4 G groups of the G smallest tiles are
// merged in registers.  The G smallest groups always lie in the G smallest tiles: a group g
// outside them would have G tiles, each holding a group with (minimum, index) below g's, before it.
template <int CAP>
__device__ __forceinline__ uint64_t topg_select_row(const float* __restrict__ g, int n, int G,
                                                    const float* __restrict__ fine, int n_fine, uint64_t* buf,
                                                    int lane) {
    constexpr int FINE_PER = 4;
    static_assert(CAP >= 32 && (CAP & (CAP - 1)) == 0, "the sorted buffer is a power of two >= 32");
    // (n <= 512, the usual case -- 65 536 lists = 512 tiles: the row is loaded ONCE, 16 independent
    // loads per lane, and both passes run on registers; the loops below were bound by one L2
    // latency per iteration)
    constexpr int REGV = 16;
    const bool in_regs = n <= 32 * REGV;
    float rv[REGV];
    if (in_regs) {
#pragma unroll
        for (int i = 0; i < REGV; i++) {
            const int j = lane + 32 * i;
            rv[i] = (j < n) ? g[j] : 0.f;
        }
    }
    // 1. lane minima -> bound
    uint64_t lmin = DFX_COMP_NONE;
    if (in_regs) {
#pragma unroll
        for (int i = 0; i < REGV; i++) {
            const int j = lane + 32 * i;
            const uint64_t c = (j < n) ? dfx_comp(rv[i], (uint32_t)j) : DFX_COMP_NONE;
            lmin = c < lmin ? c : lmin;
        }
    } else {
        for (int j = lane; j < n; j += 32) {
            const uint64_t c = dfx_comp(g[j], (uint32_t)j);
            lmin = c < lmin ? c : lmin;
        }
    }
    const uint64_t x = dfx_warp_sort32_asc(lmin, lane);  // the 32 lane minima, ascending by lane
    const uint64_t bound = __shfl_sync(0xffffffffu, x, G - 1);  // G-th smallest lane minimum
    // 2. collect everything <= bound
    int cnt = 0;
    bool overflow = false;
    auto collect = [&](int j, float gv) {  // lanes j0 .. j0 + 31 of one warp-uniform step
        const uint64_t c = (j < n) ? dfx_comp(gv, (uint32_t)j) : DFX_COMP_NONE;
        const bool want = c <= bound && c != DFX_COMP_NONE;
        const unsigned mask = __ballot_sync(0xffffffffu, want);
        if (mask) {
            const int pos = cnt + __popc(mask & ((1u << lane) - 1u));
            if (want && pos < CAP) buf[pos] = c;
            cnt += __popc(mask);
            if (cnt > CAP) overflow = true;
        }
    };
    if (in_regs) {
#pragma unroll
        for (int i = 0; i < REGV; i++)
            if (32 * i < n) collect(lane + 32 * i, rv[i]);
    } else {
        for (int j0 = 0; j0 < n; j0 += 32) collect(j0 + lane, j0 + lane < n ? g[j0 + lane] : 0.f);
    }
    if (!overflow) {
        dfx_warp_sort_buf(buf, cnt, lane);  // 3. sort the candidates (padded to >= 32 slots)
    } else {
        // fallback: G rounds of "smallest composite above the previous pick", left in buf[0..G)
        uint64_t prev = 0;
        for (int r = 0; r < G; r++) {
            uint64_t best = DFX_COMP_NONE;
            for (int j = lane; j < n; j += 32) {
                const uint64_t c = dfx_comp(g[j], (uint32_t)j);
                if ((r == 0 || c > prev) && c < best) best = c;
            }
#pragma unroll
            for (int off = 16; off >= 1; off >>= 1) {
                const uint64_t o = __shfl_xor_sync(0xffffffffu, best, off);
                best = o < best ? o : best;
            }
            if (lane == 0) buf[r] = best;
            prev = best;
            if (best == DFX_COMP_NONE) prev = DFX_COMP_NONE - 1;
        }
        __syncwarp();
    }
    uint64_t sel = lane < G ? buf[lane] : DFX_COMP_NONE;
    __syncwarp();  // buf is free again
    if (fine) {  // second level: the 32 smallest of the 4 groups of each selected tile
        uint64_t fc[FINE_PER];
#pragma unroll
        for (int j = 0; j < FINE_PER; j++) {
            const int64_t gi = (int64_t)(uint32_t)sel * FINE_PER + j;
            fc[j] = (sel != DFX_COMP_NONE && gi < n_fine) ? dfx_comp(fine[gi], (uint32_t)gi) : DFX_COMP_NONE;
        }
        sel = dfx_warp_sort32_asc(fc[0], lane);
#pragma unroll
        for (int j = 1; j < FINE_PER; j++) sel = dfx_warp_merge_sorted32(sel, dfx_warp_sort32_asc(fc[j], lane), lane);
        if (lane >= G) sel = DFX_COMP_NONE;
    }
    return sel;
}
// the selection above for a row per warp -> groups[row][0..G) (-1 = none), G <= 32
template <int CAP>
__global__ void __launch_bounds__(256)
topg_collect_kernel(const float* __restrict__ coarse, int64_t nq, int n, int G, const float* __restrict__ fine,
                    int n_fine, int32_t* __restrict__ groups) {
    __shared__ uint64_t s_buf[8][CAP];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int64_t row = (int64_t)blockIdx.x * 8 + warp;
    if (row >= nq) return;
    const uint64_t c = topg_select_row<CAP>(coarse + row * n, n, G, fine ? fine + row * n_fine : nullptr, n_fine,
                                            s_buf[warp], lane);
    if (lane < G) groups[row * G + lane] = (c == DFX_COMP_NONE) ? -1 : (int32_t)(uint32_t)c;
}
// exact canonical fp32 values of the candidates.
//   MODE 0: out[row][c] = comp(value, centroid) for every candidate slot (NONE for unused slots)
//   MODE 1: write the arg-min centroid to assign[row]
//   MODE 2: select the nprobe smallest in shared memory and write keys[row][0..nprobe) (sorted)
// rows: optional indirection (the CTA for list entry b handles row rows[b]); nrows_dev: its length.
// T: the table's row type, float, or __half for the stored rows of FLAT_SQ16 (MODE 0)
template <int MODE, class T = float>
__global__ void __launch_bounds__(128)
rerank_kernel(const float* __restrict__ Q, int d, const T* __restrict__ cent, const float* __restrict__ cnorm,
              int64_t nlist, int metric, const int32_t* __restrict__ groups, int G, int nprobe,
              const float* __restrict__ gmin, const float* __restrict__ gmin2, const uint8_t* __restrict__ gargc,
              int ng, ScreenTol tol, uint64_t* __restrict__ out, int32_t* __restrict__ assign,
              const int32_t* __restrict__ rows, const int32_t* __restrict__ nrows_dev, int64_t nrows,
              int32_t* __restrict__ keys, int32_t* __restrict__ ovf) {
    DFX_DYN_SMEM(unsigned char, rr_smem, 16);
    float* s_q = reinterpret_cast<float*>(rr_smem);
    uint64_t* s_c = reinterpret_cast<uint64_t*>(rr_smem + ((size_t)d * 4 + 15) / 16 * 16);  // MODE 2
    __shared__ unsigned long long s_best[4];
    __shared__ float s_thr;
    __shared__ int s_cnt;
    const int ncand = G * 32;
    const int64_t limit = nrows_dev ? (int64_t)*nrows_dev : nrows;
    for (int64_t b = blockIdx.x; b < limit; b += gridDim.x) {
        const int64_t row = rows ? rows[b] : b;
        __syncthreads();
        for (int i = threadIdx.x; i < d; i += 128) s_q[i] = Q[row * d + i];
        if (threadIdx.x == 0) s_cnt = 0;
        __syncthreads();
        if (threadIdx.x == 0) s_thr = screen_threshold(groups, row, G, nprobe, ng, gmin, tol, ovf);
        __syncthreads();
        const float thr = s_thr;
        unsigned long long best = DFX_COMP_NONE;
        for (int c = threadIdx.x; c < ncand; c += 128) {
            const int gid = groups[row * G + (c >> 5)];
            unsigned long long comp = DFX_COMP_NONE;
            if (gid >= 0) {
                const int64_t o = row * ng + gid;
                bool expand;
                const bool live = group_live(gmin[o], gmin2[o], thr, expand) && (expand || (c & 31) == (int)gargc[o]);
                const int64_t col = (int64_t)gid * 32 + (c & 31);
                if (live && col < nlist)
                    comp = dfx_comp(dfx_rank_value(dfx_dot_seqk(s_q, cent + col * d, d), metric, cnorm, col),
                                    (uint32_t)col);
            }
            if (MODE == 1) best = comp < best ? comp : best;
            else if (MODE == 0) out[row * ncand + c] = comp;
            else if (comp != DFX_COMP_NONE) s_c[atomicAdd(&s_cnt, 1)] = comp;
        }
        if (MODE == 1) {
#pragma unroll
            for (int off = 16; off >= 1; off >>= 1) {
                unsigned long long o = __shfl_xor_sync(0xffffffffu, best, off);
                best = o < best ? o : best;
            }
            if ((threadIdx.x & 31) == 0) s_best[threadIdx.x >> 5] = best;
            __syncthreads();
            if (threadIdx.x == 0) {
                for (int w = 1; w < 4; w++) best = s_best[w] < best ? s_best[w] : best;
                assign[row] = (best == DFX_COMP_NONE) ? -1 : (int32_t)(uint32_t)best;
            }
        }
        if (MODE == 2) {
            __syncthreads();
            const int cnt = s_cnt;
            int P = 32;
            while (P < cnt) P <<= 1;
            for (int e = cnt + threadIdx.x; e < P; e += 128) s_c[e] = DFX_COMP_NONE;
            dfx_block_bitonic_sort<128>(s_c, P);
            for (int j = threadIdx.x; j < nprobe; j += 128) {
                const uint64_t c = (j < P) ? s_c[j] : DFX_COMP_NONE;
                keys[row * nprobe + j] = (c == DFX_COMP_NONE) ? -1 : (int32_t)(uint32_t)c;
            }
        }
    }
}

// ---- the exact re-rank of a row by one warp (decide_rows_kernel): lanes own the
// selected groups, live candidates are compacted into a per-warp list (arg-min column, or all 32
// columns of a group whose runner-up is within the tolerance), each lane evaluates one candidate
// in the canonical seq-k order, and the nprobe smallest come out of a register bitonic network.
// The candidate set is a superset of the true top-nprobe for any tolerance >= the screening error,
// so the keys are identical to rerank_kernel<2>'s.
// Appends this step's 32 groups (gid -1 = none; live / expand per group_live, argc = the arg-min
// column) to s_cand[cnt ..), returns the new count.
__device__ __forceinline__ int decide_add_candidates(int gid, bool live, bool expand, int argc, int64_t nlist,
                                                     int32_t* __restrict__ s_cand, int cnt, int lane) {
    expand = live && expand;
    const bool single = live && !expand && ((int64_t)gid * 32 + argc) < nlist;
    const unsigned ms = __ballot_sync(0xffffffffu, single);
    if (single) s_cand[cnt + __popc(ms & ((1u << lane) - 1u))] = gid * 32 + argc;
    cnt += __popc(ms);
    unsigned me = __ballot_sync(0xffffffffu, expand);
    while (me) {  // rare: a group whose runner-up cannot be ruled out contributes all its columns
        const int src = __ffs((int)me) - 1;
        me &= me - 1;
        const int eg = __shfl_sync(0xffffffffu, gid, src);
        const int64_t col = (int64_t)eg * 32 + lane;
        const bool ok = col < nlist;
        const unsigned mo = __ballot_sync(0xffffffffu, ok);
        if (ok) s_cand[cnt + __popc(mo & ((1u << lane) - 1u))] = (int32_t)col;
        cnt += __popc(mo);
    }
    return cnt;
}
// exact canonical values of the cnt candidates, 32 at a time; keys_row[0 .. nprobe) = the
// nprobe (<= 32) smallest, ascending (-1 = none)
__device__ __forceinline__ void decide_exact_keys(const float* __restrict__ s_q, int d, const float* __restrict__ cent,
                                                  const float* __restrict__ cnorm, int metric,
                                                  const int32_t* __restrict__ s_cand, int cnt, int nprobe,
                                                  int32_t* __restrict__ keys_row, int lane) {
    __syncwarp();
    uint64_t kept = DFX_COMP_NONE;
    for (int c0 = 0; c0 < cnt; c0 += 32) {
        uint64_t comp = DFX_COMP_NONE;
        if (c0 + lane < cnt) {
            const int64_t col = s_cand[c0 + lane];
            comp = dfx_comp(dfx_rank_value(dfx_dot_seqk(s_q, cent + col * d, d), metric, cnorm, col), (uint32_t)col);
        }
        kept = dfx_warp_merge_sorted32(kept, dfx_warp_sort32_asc(comp, lane), lane);
    }
    if (lane < nprobe) keys_row[lane] = (kept == DFX_COMP_NONE) ? -1 : (int32_t)(uint32_t)kept;
}

// Search path, nprobe <= 32 and G <= 64: the decide stage of a row by one warp, from the
// screening summary to the keys.  LEVELS says where the row's groups come from:
//   2: topg_select_row on the tile minima, then on gmin (G <= 32 of ng >= 128; the bench shape);
//   1: topg_select_row on gmin alone (G <= 32 of 32 <= ng < 128);
//   0: given in groups[row][0 .. G), from tc_select_groups (33 <= G <= 64).
// A selection in the kernel leaves lane r with the r-th smallest selected group; the group's
// minimum is the value of its composite, so the threshold, the overflow test and the liveness of
// a group need no load; only the runner-up and the arg-min column of the selected groups are
// read, together with the query row.  Nothing goes through global memory between the selection
// and the re-rank.  Given groups are walked in slices of 32, one per lane.
// Per warp: the selection buffer (later the candidate list), then the row's query.  Warps per
// CTA: 8, or 4 on given groups, where 8 took 4-9 % longer at 2048 lists (4096 queries, d = 128,
// H100 80GB HBM3 at 700 W).
constexpr int DECIDE_CAP = 256;
__host__ __device__ constexpr int decide_warps(int levels) { return levels > 0 ? 8 : 4; }
__host__ __device__ __forceinline__ size_t decide_slots(int G) {  // bytes: DECIDE_CAP composites or G x 32 columns
    return (size_t)DECIDE_CAP * 8 > (size_t)G * 32 * 4 ? (size_t)DECIDE_CAP * 8 : (size_t)G * 32 * 4;
}
static size_t decide_rows_smem(int d, int G, int warps) {
    return warps * (decide_slots(G) + (size_t)(d + 3) / 4 * 4 * 4);
}
template <int LEVELS>
__global__ void __launch_bounds__(decide_warps(LEVELS) * 32)
decide_rows_kernel(const float* __restrict__ Q, int d, const float* __restrict__ cent,
                   const float* __restrict__ cnorm, int64_t nlist, int metric, const float* __restrict__ tmin,
                   const float* __restrict__ gmin, const float* __restrict__ gmin2,
                   const uint8_t* __restrict__ gargc, int ng, int G, int nprobe, ScreenTol tol, int64_t nrows,
                   int32_t* __restrict__ keys, int32_t* __restrict__ ovf, const int32_t* __restrict__ groups) {
    DFX_DYN_SMEM(unsigned char, dr_smem, 16);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int64_t row = (int64_t)blockIdx.x * decide_warps(LEVELS) + warp;
    if (row >= nrows) return;  // whole warps leave; no block-wide barrier below
    const size_t slots = decide_slots(G);
    unsigned char* own = dr_smem + (size_t)warp * (slots + (size_t)(d + 3) / 4 * 4 * 4);
    uint64_t* buf = reinterpret_cast<uint64_t*>(own);
    int32_t* s_cand = reinterpret_cast<int32_t*>(own);  // once the selection is done with buf
    float* s_q = reinterpret_cast<float*>(own + slots);
    const int nt = ng / 4;
    uint64_t sel = DFX_COMP_NONE;
    if constexpr (LEVELS == 2) sel = topg_select_row<DECIDE_CAP>(tmin + row * nt, nt, G, gmin + row * ng, ng, buf, lane);
    if constexpr (LEVELS == 1) sel = topg_select_row<DECIDE_CAP>(gmin + row * ng, ng, G, nullptr, 0, buf, lane);
    const int gid = (sel == DFX_COMP_NONE) ? -1 : (int32_t)(uint32_t)sel;
    float m2 = 0.f;
    int argc = 0;
    if (gid >= 0) {
        m2 = gmin2[row * ng + gid];
        argc = (int)gargc[row * ng + gid];
    }
    for (int i = lane; i < d; i += 32) s_q[i] = Q[row * d + i];
    float thr = 0.f;
    int cnt = 0;
    if constexpr (LEVELS == 0) {
        if (lane == 0) thr = screen_threshold(groups, row, G, nprobe, ng, gmin, tol, ovf);
        thr = __shfl_sync(0xffffffffu, thr, 0);
        for (int g0 = 0; g0 < G; g0 += 32) {
            const int gg = g0 + lane < G ? groups[row * G + g0 + lane] : -1;
            bool live = false, expand = false;
            int ac = 0;
            if (gg >= 0) {
                const int64_t o = row * ng + gg;
                live = group_live(gmin[o], gmin2[o], thr, expand);
                ac = (int)gargc[o];
            }
            cnt = decide_add_candidates(gg, live, expand, ac, nlist, s_cand, cnt, lane);
        }
    } else {
        // gmin of the lane's group (dfx_key2f gives back gmin + 0: -0 reads as +0, which no
        // comparison below tells apart); t and last as screen_threshold(groups, ...) defines them
        const float nan = __int_as_float(0x7fc00000), inf = __int_as_float(0x7f800000);
        const float m1 = (gid >= 0) ? dfx_key2f((uint32_t)(sel >> 32)) : nan;
        const float tk = __shfl_sync(0xffffffffu, gid >= 0 ? m1 : inf, nprobe <= G ? nprobe - 1 : 0);
        const float tl = __shfl_sync(0xffffffffu, m1, G - 1);
        if (lane == 0) thr = screen_threshold(nprobe <= G ? tk : inf, G < ng ? tl : nan, row, tol, ovf);
        thr = __shfl_sync(0xffffffffu, thr, 0);
        bool expand = false;
        const bool live = gid >= 0 && group_live(m1, m2, thr, expand);
        cnt = decide_add_candidates(gid, live, expand, argc, nlist, s_cand, 0, lane);
    }
    decide_exact_keys(s_q, d, cent, cnorm, metric, s_cand, cnt, nprobe, keys + row * nprobe, lane);
}
// assign fast path: one thread per row decides from the screening summary alone when the best
// group's arg-min column is unambiguous (no other column within tol); other rows are queued
// for the exact evaluation above.
__global__ void assign_resolve_kernel(const int32_t* __restrict__ groups, const float* __restrict__ gmin,
                                      const float* __restrict__ gmin2, const uint8_t* __restrict__ gargc, int ng,
                                      int G, ScreenTol tol, int64_t n, int32_t* __restrict__ assign,
                                      int32_t* __restrict__ amb_rows, int32_t* __restrict__ amb_count,
                                      int32_t* __restrict__ ovf) {
    const int64_t row = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (row >= n) return;
    const int g0 = groups[row * G + 0], g1 = (G > 1) ? groups[row * G + 1] : -1;
    const int64_t o0 = row * ng + g0;
    const float thr = gmin[o0] + screen_tol(tol, row, tol.rel);
    if (tol.rel_fast > 0.f && screen_last_min(groups, row, G, ng, gmin) <= gmin[o0] + screen_tol(tol, row, tol.rel_fast))
        atomicAdd(&ovf[1], 1);  // AUTO mode statistic: FAST would send this row to the exact fallback
    const bool clear = gmin2[o0] > thr && (g1 < 0 || gmin[row * ng + g1] > thr);
    if (clear) {
        assign[row] = g0 * 32 + (int)gargc[o0];
    } else {
        assign[row] = -1;
        amb_rows[atomicAdd(amb_count, 1)] = (int32_t)row;
    }
}

// ---- exact fallback for the rows the decide stage flagged (screen_overflow): the K smallest
// composites over ALL columns, canonical values computed on the fly (seq-k FMA, the same chain as
// rerank_kernel), selected by the radix select of dfx_select.cuh.  Rare by construction (more than
// `margin` group minima within the tolerance: duplicate centroids / duplicate rows); slow but exact.
template <class T>  // the table's row type (rerank_kernel)
struct ExactLoader {
    const float* q;  // the row's query, staged in shared memory by the kernel
    const T* X;
    const float* xnorm;
    int d, metric;   // d % 4 == 0 (the tensor-core path requires d % 64 == 0)
    __device__ __forceinline__ uint64_t operator()(int64_t /*row*/, int e) const {
        return dfx_comp(dfx_rank_value(dfx_dot_seqk(q, X + (int64_t)e * d, d), metric, xnorm, e), (uint32_t)e);
    }
};
struct ExactWriter {  // mode 2: keys[row][K]; mode 1: assign[row]; mode 0: out[row][K] composites
    int mode, K;
    int32_t* keys;
    int32_t* assign;
    uint64_t* out;
    __device__ __forceinline__ void operator()(int64_t row, int j, uint64_t c) const {
        const int32_t col = (c == DFX_COMP_NONE) ? -1 : (int32_t)(uint32_t)c;
        if (mode == 2) keys[row * K + j] = col;
        else if (mode == 1) assign[row] = col;
        else out[row * K + j] = c;
    }
};
// dynamic smem: P composites, then the row's query (d floats)
template <class T>
__global__ void __launch_bounds__(256)
tc_exact_rows_kernel(const float* __restrict__ Q, ExactLoader<T> ld, ExactWriter wr, const int32_t* __restrict__ ovf,
                     int n, int k, int P, int sort_cap) {
    DFX_DYN_SMEM(unsigned char, ex_smem, 16);
    uint64_t* s_out = reinterpret_cast<uint64_t*>(ex_smem);
    float* s_q = reinterpret_cast<float*>(ex_smem + (size_t)P * 8);
    ld.q = s_q;
    const int count = ovf[0];
    for (int b = blockIdx.x; b < count; b += gridDim.x) {
        const int64_t row = ovf[2 + b];
        for (int i = threadIdx.x; i < ld.d; i += 256) s_q[i] = Q[row * ld.d + i];
        __syncthreads();
        dfx_select_row<256>(ld, wr, row, n, k, P, sort_cap, s_out);
        __syncthreads();
    }
}
// mode / K as in ExactWriter; Q rows are indexed by the values in ovf (chunk-relative)
template <class T>
static void launch_exact_rows(const float* Q, const T* X, const float* xnorm, int64_t ncols, int d, int metric,
                              const int32_t* ovf, int64_t nrows, int mode, int K, int32_t* keys, int32_t* assign,
                              uint64_t* out, cudaStream_t st) {
    DFX_REQUIRE(K >= 1 && K <= 4096 && ncols < (1ll << 31), "exact fallback: bad K / column count");
    const int sort_cap = 2048, n = (int)ncols;
    const int base = (n <= sort_cap) ? (n > K ? n : K) : K;
    const int P = dfx_next_pow2(base < 2 ? 2 : base);
    ExactLoader<T> ld{nullptr, X, xnorm, d, metric};
    ExactWriter wr{mode, K, keys, assign, out};
    const unsigned grid = (unsigned)std::min<int64_t>(nrows, 2 * dfx_num_sms());
    const size_t smem = (size_t)P * 8 + (size_t)d * 4;
    auto kern = tc_exact_rows_kernel<T>;
    DFX_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    DFX_LAUNCH(kern, grid, 256, smem, st, Q, ld, wr, ovf, n, K, P, sort_cap);
}

// ------------------------------------------------------------------ host side
#ifndef DFX_EMU
typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                    const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                    CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static PFN_encodeTiled get_encode_fn() {
    static PFN_encodeTiled fn = nullptr;
    if (!fn) {
        void* p = nullptr;
        cudaDriverEntryPointQueryResult qres;
        DFX_CUDA(cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres));
        DFX_REQUIRE(p != nullptr && qres == cudaDriverEntryPointSuccess, "cuTensorMapEncodeTiled not available");
        fn = (PFN_encodeTiled)p;
    }
    return fn;
}

// fp16 matrix [rows, d] row-major, box = 128 rows x 64 columns, 128-byte swizzle
static void make_tmap(CUtensorMap* tm, const void* base, int64_t rows, int d, int box_rows = tc::TILE) {
    cuuint64_t gdim[2] = {(cuuint64_t)d, (cuuint64_t)rows};
    cuuint64_t gstr[1] = {(cuuint64_t)d * 2};
    cuuint32_t box[2] = {(cuuint32_t)tc::KATOM, (cuuint32_t)box_rows};
    cuuint32_t estr[2] = {1, 1};
    CUresult r = get_encode_fn()(tm, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, const_cast<void*>(base), gdim, gstr, box,
                                 estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                                 CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    DFX_REQUIRE(r == CUDA_SUCCESS, "cuTensorMapEncodeTiled failed with code " + std::to_string((int)r));
}

#endif  // !DFX_EMU

// d = a whole number of 64-element k-atoms (d <= 256: query tile resident; above: streamed)
bool dfx_tc_supported(int d) { return d >= 64 && d % 64 == 0 && d <= 2048; }

// the screening table of rows x [n][d] (centroids / FLAT rows), synchronises: their mean m, the
// column terms, the norm maxima, and the fp16 hi and lo planes of x - m (either precision can use
// them), scaled so that the largest centred row norm lands in [2^13, 2^14)
static void tc_prepare_table(const float* x, int64_t n, int d, int metric, dfx_tc_table& tab, cudaStream_t st) {
    const int64_t n_pad = dfx_ceil_div(n, tc::TILE) * tc::TILE;
    tab.mean.reserve((size_t)d * 4 + 8 + (size_t)MEAN_CHUNKS * d * 8);
    float* mean = tab.mean.as<float>();
    float* maxima = mean + d;                                  // [2]
    double* part = reinterpret_cast<double*>(maxima + 2);      // d % 64 == 0: 8-byte aligned
    DFX_LAUNCH(col_part_kernel, dim3((unsigned)(d / 32), MEAN_CHUNKS), 256, 0, st, x, n, d, part);
    DFX_LAUNCH(col_mean_kernel, (unsigned)dfx_ceil_div(d, 128), 128, 0, st, part, d, n, mean);
    tab.cterm.reserve((size_t)n_pad * 4);
    DFX_CUDA(cudaMemsetAsync(maxima, 0, 8, st));
    DFX_LAUNCH(table_terms_kernel, (unsigned)dfx_ceil_div(n_pad, 8), 256, 0, st, x, n, n_pad, d, mean, metric,
               tab.cterm.as<float>(), maxima);
    float h[2] = {0.f, 0.f};
    DFX_CUDA(cudaMemcpyAsync(h, maxima, 8, cudaMemcpyDeviceToHost, st));
    DFX_CUDA(cudaStreamSynchronize(st));
    tab.cmax2 = h[0];
    tab.cmax2c = h[1];
    tab.scale = dfx_pow2_scale(sqrtf(tab.cmax2c));
    tab.planes.reserve((size_t)2 * n_pad * d * 2);
    DFX_LAUNCH(f16_rows_kernel, (unsigned)dfx_ceil_div(n_pad, 8), 256, 0, st, x, n, n_pad, d, (const float*)mean, 0,
               tab.scale, 0.f, 2, tab.planes.as<__half>(), (float*)nullptr, (float2*)nullptr, (float*)nullptr);
}

// install the index's screening table (its centroids, or the rows of a FLAT index); AUTO starts
// PRECISE on a new table
static void tc_install_table(dfx_index* idx, const float* x, int64_t n, cudaStream_t st) {
    tc_prepare_table(x, n, idx->cfg.d, idx->cfg.metric, idx->tc_tab, st);
    if (idx->tc_mode == 0) idx->tc_fast = false;
    idx->tc_stat_pending = false;
    idx->tc_acc_rows = idx->tc_acc_bad = 0;
}

// (re)build the screening table of the centroids; call after training / import
void dfx_tc_prepare_centroids(dfx_index* idx, cudaStream_t st) {
    if (!dfx_tc_supported(idx->cfg.d)) return;
    tc_install_table(idx, idx->centroids.as<float>(), idx->cfg.nlist, st);
    idx->tc_ready = true;
}

// ---- AUTO precision: statistics of a past launch come back through pinned memory, no sync
static bool tc_stream_capturing(cudaStream_t st) {
    cudaStreamCaptureStatus cs = cudaStreamCaptureStatusNone;
    if (cudaStreamIsCapturing(st, &cs) != cudaSuccess) {
        cudaGetLastError();
        return false;
    }
    return cs != cudaStreamCaptureStatusNone;
}
// AUTO rule.  A row that overflows costs an exact pass over ALL columns by one CTA (milliseconds
// at nlist = 65 536), more than FAST saves on a whole launch, so FAST is only worth it where
// overflows practically never happen: PRECISE -> FAST after at least 16 384 observed rows none of
// which would have overflowed under FAST's tolerance; FAST -> PRECISE as soon as more than one row
// in 16 384 did overflow.  Counts accumulate across launches (a batch of one query says nothing
// on its own).  Either way the results are exact; only the cost moves.
// Folds the counts of one launch of precision `fast` into (acc_rows, acc_bad) and returns the
// precision of the next launch; a decision starts a new window.
static bool tc_auto_step(bool fast, int64_t rows, int64_t overflowed, int64_t fast_would, int64_t window,
                         int64_t& acc_rows, int64_t& acc_bad) {
    acc_rows += rows;
    acc_bad += fast ? overflowed : fast_would;
    if (!fast && acc_rows >= window) {
        fast = acc_bad == 0;
        acc_rows = acc_bad = 0;
    } else if (fast && acc_bad > 0 && acc_bad * window > acc_rows) {
        fast = false;
        acc_rows = acc_bad = 0;
    }
    return fast;
}
// The search-path AUTO state of an index.  A switch bumps `generation` (captured graphs are stale).
static void tc_auto_update(dfx_index* idx, bool was_fast, int64_t rows, int64_t overflowed, int64_t fast_would) {
    if (idx->tc_mode != 0 || rows <= 0 || was_fast != idx->tc_fast) return;
    // window: 16 384 rows unless dfx_set_param("tc_auto_window") says otherwise
    const bool fast = tc_auto_step(was_fast, rows, overflowed, fast_would, idx->tc_auto_window, idx->tc_acc_rows,
                                   idx->tc_acc_bad);
    if (fast && idx->tc_acc_rows >= (1 << 20)) idx->tc_acc_rows = idx->tc_acc_bad = 0;  // a fresh window
    if (fast != idx->tc_fast) {
        idx->tc_fast = fast;
        idx->generation++;
    }
}
static void tc_stats_poll(dfx_index* idx, cudaStream_t st) {  // before choosing the precision of a launch
    if (!idx->tc_stat_pending || tc_stream_capturing(st)) return;  // (no event queries inside a capture)
    if (cudaEventQuery(idx->tc_stat_ev) != cudaSuccess) {
        cudaGetLastError();  // not ready yet: keep the current precision
        return;
    }
    idx->tc_stat_pending = false;
    idx->tc_last_rows = idx->tc_stat_rows;
    idx->tc_last_overflow = idx->tc_stat_h[0];
    idx->tc_last_fast_would = idx->tc_stat_h[1];
    tc_auto_update(idx, idx->tc_stat_fast, idx->tc_stat_rows, idx->tc_stat_h[0], idx->tc_stat_h[1]);
}
void dfx_tc_stats_sync(dfx_index* idx) {
    if (!idx->tc_stat_pending) return;
    cudaEventSynchronize(idx->tc_stat_ev);
    tc_stats_poll(idx, nullptr);
}
static void tc_stats_post(dfx_index* idx, const int32_t* ovf, int64_t rows, bool fast, cudaStream_t st) {
    if (idx->tc_mode != 0 || idx->tc_stat_pending || tc_stream_capturing(st)) return;
    if (!idx->tc_stat_h) {
        DFX_CUDA(cudaMallocHost(reinterpret_cast<void**>(&idx->tc_stat_h), 8));
        DFX_CUDA(cudaEventCreateWithFlags(&idx->tc_stat_ev, cudaEventDisableTiming));
    }
    DFX_CUDA(cudaMemcpyAsync(idx->tc_stat_h, ovf, 8, cudaMemcpyDeviceToHost, st));
    DFX_CUDA(cudaEventRecord(idx->tc_stat_ev, st));
    idx->tc_stat_pending = true;
    idx->tc_stat_fast = fast;
    idx->tc_stat_rows = rows;
}
// the tolerance of a launch against table `tab`, for the rows tc_screen last prepared
static ScreenTol tc_tol(const dfx_index* idx, const dfx_tc_table& tab, int d, bool fast) {
    ScreenTol t;
    t.rel = screen_tol_rel(d, fast, tab.one_plane());
    t.rel_fast = (!fast && idx->tc_mode == 0) ? screen_tol_rel(d, true, tab.one_plane()) : 0.f;
    t.raw = screen_tol_raw(d);
    t.cmax2 = tab.cmax2;
    t.cmax2c = tab.cmax2c;
    t.qn = idx->tc_qn.as<float2>();
    return t;
}

// screening pass: gmin[nq][ng] for a batch of rows against a table prepared by tc_prepare_table
// (npl planes used); leaves the rows' norms in idx->tc_qn
static void tc_screen(dfx_index* idx, int d, const float* d_x, int64_t nq, const dfx_tc_table& tab, int npl,
                      int64_t nlist, int metric, float* gmin, float* gmin2, uint8_t* gargc, float* tmin,
                      cudaStream_t st) {
    using namespace tc;
    const int64_t nl_pad = dfx_ceil_div(nlist, TILE) * TILE;
    const int64_t nq_pad = dfx_ceil_div(nq, TILE) * TILE;
    const int ng = (int)(nl_pad / 32);
    idx->tc_q.reserve((size_t)npl * nq_pad * d * 2);
    idx->tc_qmult.reserve((size_t)nq_pad * 4);
    idx->tc_qterm.reserve((size_t)nq_pad * 4);
    idx->tc_qn.reserve((size_t)nq_pad * 8);
    DFX_LAUNCH(f16_rows_kernel, (unsigned)dfx_ceil_div(nq_pad, 8), 256, 0, st, d_x, nq, nq_pad, d,
               (const float*)tab.mean.as<float>(), 1, tab.scale, metric == DFX_METRIC_IP ? -1.f : -2.f, npl,
               idx->tc_q.as<__half>(), idx->tc_qmult.as<float>(), idx->tc_qn.as<float2>(), idx->tc_qterm.as<float>());
    // one exact plane: the stored rows themselves, nlist of them (TMA zero-fills the last tile's tail)
    const bool one = tab.one_plane();
    const void* table_h = one ? static_cast<const void*>(tab.rows) : tab.planes.p;
    const float* cterm = one ? tab.rows_cterm : tab.cterm.as<float>();
#ifdef DFX_EMU
    emu_tc_screen(idx->tc_q.as<__half>(), idx->tc_qmult.as<float>(), idx->tc_qterm.as<float>(), nq, nq_pad,
                  static_cast<const __half*>(table_h), nl_pad, nlist, one, d, npl, cterm, gmin, gmin2, gargc, tmin,
                  ng);
    return;
#else
    const int katoms = d / KATOM;
    // resident only for the k-atom counts the kernel is instantiated for (1, 2, 4); others stream
    const bool res = Smem::resident(katoms, npl) && (katoms == 1 || katoms == 2 || katoms == 4);
    CUtensorMap tmQ, tmC;
    make_tmap(&tmQ, idx->tc_q.p, npl * nq_pad, d);
    make_tmap(&tmC, table_h, one ? nlist : npl * nl_pad, d);
    const int qtiles = (int)(nq_pad / TILE), ctiles = (int)(nl_pad / TILE);
    const size_t smem = (size_t)Smem::total(res, katoms, npl) + 1024;
    const int slots = dfx_num_sms() * Smem::ctas_per_sm(res, katoms, npl);  // CTAs resident at once
    // split the centroid tiles so that the grid is close to a whole number of waves while every
    // CTA keeps enough tiles to amortise its start (query tile, pipeline fill):
    // cost model = waves x (tiles per CTA + ~3 tiles of fixed overhead)
    int csplit = 1, per = ctiles;
    {
        double best_cost = 1e30;
        for (int cs = 1; cs <= ctiles && cs <= 4096; cs++) {
            const int pr = (int)dfx_ceil_div(ctiles, cs);
            const int cs_eff = (int)dfx_ceil_div(ctiles, pr);
            if (cs_eff != cs) continue;
            const int64_t ctas = (int64_t)qtiles * cs;
            const double waves = (double)dfx_ceil_div(ctas, slots);
            const double cost = waves * (pr + 3.0);
            if (cost < best_cost - 1e-9) {
                best_cost = cost;
                csplit = cs;
                per = pr;
            }
        }
    }
    dim3 grid((unsigned)csplit, (unsigned)qtiles);
    DFX_REQUIRE(qtiles <= 65535, "too many query tiles in one screening launch");
#define DFX_TC_LAUNCH(KT_, NP, ONE_)                                                                     \
    do {                                                                                                 \
        auto kern = tc_coarse_kernel<KT_, NP, ONE_>;                                                     \
        DFX_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));    \
        DFX_LAUNCH(kern, grid, THREADS, smem, st, tmQ, tmC, (int)nq, (int)nq_pad, (int)nl_pad, (int)nlist, katoms, \
                   cterm, idx->tc_qmult.as<float>(), idx->tc_qterm.as<float>(), per, gmin, gmin2, gargc, tmin, ng); \
    } while (0)
    // resident shapes get their k-atom count at compile time (npl * katoms <= 4); FAST takes either table
    if (npl == 1) {
        if (res && katoms == 1) DFX_TC_LAUNCH(1, 1, false);
        else if (res && katoms == 2) DFX_TC_LAUNCH(2, 1, false);
        else if (res && katoms == 4) DFX_TC_LAUNCH(4, 1, false);
        else DFX_TC_LAUNCH(0, 1, false);
    } else if (one) {
        if (res && katoms == 1) DFX_TC_LAUNCH(1, 2, true);
        else if (res && katoms == 2) DFX_TC_LAUNCH(2, 2, true);
        else DFX_TC_LAUNCH(0, 2, true);
    } else {
        if (res && katoms == 1) DFX_TC_LAUNCH(1, 2, false);
        else if (res && katoms == 2) DFX_TC_LAUNCH(2, 2, false);
        else DFX_TC_LAUNCH(0, 2, false);
    }
#undef DFX_TC_LAUNCH
#endif  // DFX_EMU
}

// the G groups of every row with the smallest minima, ascending: two-level warp selection for
// G <= 32 (tile minima first), the generic radix select otherwise
static void tc_select_groups(const float* gmin, const float* tmin, int64_t nrows, int ng, int G, int32_t* groups,
                             cudaStream_t st) {
    if (G <= 32 && ng >= 128) {
        auto tk = topg_collect_kernel<256>;
        DFX_LAUNCH(tk, (unsigned)dfx_ceil_div(nrows, 8), 256, 0, st, tmin, nrows, ng / 4, G, gmin, ng, groups);
    } else if (G <= 32 && ng >= 32) {
        auto tk = topg_collect_kernel<256>;
        DFX_LAUNCH(tk, (unsigned)dfx_ceil_div(nrows, 8), 256, 0, st, gmin, nrows, ng, G, (const float*)nullptr, 0,
                   groups);
    } else {
        dfx_launch_select_cols(gmin, nrows, ng, ng, G, 0, groups, nullptr, nullptr, 0, st);
    }
}

// what the decide stage reads: the screening summary [rows][ng] and its tile minima
// [rows][ng / 4], the G selected groups per row (when asked for), and the overflow record
// [overflow rows, FAST-would-overflow rows, row list ...], zeroed
struct Screened {
    const float* gmin;
    const float* gmin2;
    const uint8_t* gargc;
    const float* tmin;
    const int32_t* groups;
    int32_t* ovf;
};
// screen a chunk of `rows` rows against a table (as tc_screen), then, for G > 0, select the G
// groups of every row into tc_groups; the workspace is sized for chunks of up to rmax rows
static Screened tc_screen_chunk(dfx_index* idx, int d, const float* d_x, int64_t rows, int64_t rmax, int ng, int G,
                                const dfx_tc_table& tab, int npl, int64_t nlist, int metric, cudaStream_t st) {
    idx->tc_gmin.reserve((size_t)rmax * ng * 4);
    idx->tc_gmin2.reserve((size_t)rmax * ng * 4);
    idx->tc_gargc.reserve((size_t)rmax * ng);
    idx->tc_tmin.reserve((size_t)rmax * (ng / 4 + 1) * 4);
    float* gmin = idx->tc_gmin.as<float>();
    float* tmin = idx->tc_tmin.as<float>();
    tc_screen(idx, d, d_x, rows, tab, npl, nlist, metric, gmin, idx->tc_gmin2.as<float>(), idx->tc_gargc.as<uint8_t>(),
              tmin, st);
    idx->tc_ovf.reserve((size_t)(rows + 2) * 4);
    DFX_CUDA(cudaMemsetAsync(idx->tc_ovf.p, 0, 8, st));
    int32_t* groups = nullptr;
    if (G > 0) {
        idx->tc_groups.reserve((size_t)rmax * G * 4);
        groups = idx->tc_groups.as<int32_t>();
        tc_select_groups(gmin, tmin, rows, ng, G, groups, st);
    }
    return {gmin, idx->tc_gmin2.as<float>(), idx->tc_gargc.as<uint8_t>(), tmin, groups, idx->tc_ovf.as<int32_t>()};
}

// the screening summary alone (dfx_debug_tc_screen): gmin / gmin2 float [nq][ng] and gargc u8
// [nq][ng], ng = ceil(nlist / 128) * 4, of nq device queries against the index's centroid table,
// at npl planes (1 FAST, 2 PRECISE)
void dfx_tc_debug_screen(dfx_index* idx, int64_t nq, const float* d_x, int npl, float* gmin, float* gmin2,
                         uint8_t* gargc, cudaStream_t st) {
    DFX_REQUIRE(idx->tc_ready, "the index has no tensor-core screening table (untrained, or d not a multiple of 64)");
    const int64_t nlist = idx->cfg.nlist;
    const int ng = (int)(dfx_ceil_div(nlist, tc::TILE) * tc::TILE / 32);
    idx->tc_tmin.reserve((size_t)nq * (ng / 4) * 4);
    tc_screen(idx, idx->cfg.d, d_x, nq, idx->tc_tab, npl, nlist, idx->cfg.metric, gmin, gmin2, gargc,
              idx->tc_tmin.as<float>(), st);
}

// top-nprobe lists per query -> keys int32 [nq, nprobe] (exactly the oracle's coarse result)
void dfx_tc_coarse_search(dfx_index* idx, const float* d_x, int64_t nq, int nprobe, int32_t* keys, cudaStream_t st) {
    const int d = idx->cfg.d;
    const int64_t nlist = idx->cfg.nlist;
    const int metric = idx->cfg.metric;
    const int64_t nl_pad = dfx_ceil_div(nlist, tc::TILE) * tc::TILE;
    const int ng = (int)(nl_pad / 32);
    tc_stats_poll(idx, st);
    const bool fast = idx->tc_fast;
    // groups kept per query: nprobe + 8 at PRECISE.  FAST's tolerance is wider: where FAST is used
    // or may be chosen (AUTO, which counts FAST's overflows on PRECISE launches) up to nprobe + 24,
    // at most 32 (the two-level group selection); on the bench data nprobe + 8 left 3 rows in
    // 10 000 with more near-ties than selected groups under FAST, nprobe + 16 none.  With few
    // groups in all (nlist <= 2048) every one is kept, so that no row can overflow (at d = 768,
    // nprobe 32 of 64 groups, most rows did)
    int G = nprobe + 8;
    if (fast || idx->tc_mode == 0) G = std::max(G, std::min(32, nprobe + 24));
    if (G > ng || ng <= 64) G = ng;
    const int64_t QC = std::max<int64_t>(tc::TILE, ((64ll << 20) / ((int64_t)ng * 4)) / tc::TILE * tc::TILE);
    const int64_t qmax = std::min<int64_t>(nq, QC);
    const float* cent = idx->centroids.as<float>();
    const float* cnorm = idx->cnorm.as<float>();
    for (int64_t q0 = 0; q0 < nq; q0 += QC) {
        const int64_t qc = std::min(QC, nq - q0);
        const float* xq = d_x + q0 * d;
        int32_t* kq = keys + q0 * nprobe;
        // nprobe <= 32: the decide stage by one warp per row, on groups it selects itself where
        // topg_select_row takes the shape (G <= 32), else on those tc_select_groups selected
        const bool warp_rows = nprobe <= 32 && G <= 64 && d % 4 == 0;
        const int levels = !warp_rows || G > 32 || ng < 32 ? 0 : ng >= 128 ? 2 : 1;
        const int npl = fast ? 1 : 2;
        const Screened s = tc_screen_chunk(idx, d, xq, qc, qmax, ng, levels > 0 ? 0 : G, idx->tc_tab, npl, nlist,
                                           metric, st);
        const ScreenTol tol = tc_tol(idx, idx->tc_tab, d, fast);
        const int P_cand = dfx_next_pow2(G * 32 < 32 ? 32 : G * 32);
        if (warp_rows) {
            auto kern = levels == 2 ? decide_rows_kernel<2> : levels == 1 ? decide_rows_kernel<1> : decide_rows_kernel<0>;
            const int warps = decide_warps(levels);
            const size_t smem = decide_rows_smem(d, G, warps);
            if (smem > 48 * 1024)
                DFX_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
            DFX_LAUNCH(kern, (unsigned)dfx_ceil_div(qc, warps), warps * 32, smem, st, xq, d, cent, cnorm, nlist, metric,
                       s.tmin, s.gmin, s.gmin2, s.gargc, ng, G, nprobe, tol, qc, kq, s.ovf, s.groups);
        } else if (P_cand <= 4096) {  // fused: candidates never leave the SM
            auto kern = rerank_kernel<2>;
            const size_t smem = ((size_t)d * 4 + 15) / 16 * 16 + (size_t)P_cand * 8;
            DFX_LAUNCH(kern, (unsigned)qc, 128, smem, st, xq, d, cent, cnorm, nlist, metric, s.groups, G, nprobe,
                       s.gmin, s.gmin2, s.gargc, ng, tol, (uint64_t*)nullptr, (int32_t*)nullptr,
                       (const int32_t*)nullptr, (const int32_t*)nullptr, qc, kq, s.ovf);
        } else {
            idx->tc_cand.reserve((size_t)qmax * G * 32 * 8);
            auto kern = rerank_kernel<0>;
            DFX_LAUNCH(kern, (unsigned)qc, 128, (size_t)d * 4, st, xq, d, cent, cnorm, nlist, metric, s.groups, G,
                       nprobe, s.gmin, s.gmin2, s.gargc, ng, tol, idx->tc_cand.as<uint64_t>(),
                       (int32_t*)nullptr, (const int32_t*)nullptr, (const int32_t*)nullptr, qc, (int32_t*)nullptr,
                       s.ovf);
            dfx_launch_select_comp(idx->tc_cand.as<uint64_t>(), qc, G * 32, (int64_t)G * 32, nprobe, kq, st);
        }
        // rows with more near-ties than selected groups (screen_overflow): exact, over all lists
        launch_exact_rows(xq, cent, cnorm, nlist, d, metric, s.ovf, qc, 2, nprobe, kq, nullptr, nullptr, st);
        if (q0 + QC >= nq) tc_stats_post(idx, s.ovf, qc, fast, st);
    }
}

// Flat search on tensor cores (default for d a multiple of 64 up to 2048, N >= 1024, k <= 100; dfx_set_param
// "flat_tensor_cores" = 0 selects the FFMA GEMM; the results are bit-identical): flat search (reference
// index.py:94 IndexFlatIP, and IndexFlatL2 of the C-ABI) through the same machinery, with the
// database rows in place of the centroids and k in place of nprobe.  Screening on tensor cores
// over fp16 planes of the rows (built lazily, rebuilt after an add), the k + 8 groups with the
// smallest minima, exact canonical values of the columns the screening cannot rule out
// (rerank_kernel<0>) -- the values gemm_values_kernel would have produced for them, bit for bit.
// FLAT_SQ16 screens its stored fp16 rows as one exact plane (tc_install_rows) and re-ranks them in place.
// Leaves nq x ncand composites in idx->tc_cand and returns ncand; the caller selects and writes (D, I).
bool dfx_tc_flat_covers(const dfx_index* idx, int k) {
    return dfx_tc_supported(idx->cfg.d) && idx->n_sorted >= 1024 && k <= 100;
}

// max over fp16 rows of |x|^2 (one warp per row, fp64 sums rounded once; atomicMax on the bits of
// non-negative floats).  A non-finite code makes it +inf or NaN.
__global__ void __launch_bounds__(256)
rows_max2_kernel(const __half* __restrict__ x, int64_t n, int d, float* __restrict__ max2) {
    const int lane = threadIdx.x & 31;
    const int64_t row = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (row >= n) return;
    double n2 = 0.0;
    for (int k = lane; k < d; k += 32) {
        const double v = __half2float(x[row * d + k]);
        n2 += v * v;
    }
    n2 = tc_warp_sum(n2);
    const float r = (float)n2;
    if (lane == 0) atomicMax(reinterpret_cast<int*>(max2), __float_as_int(r <= FLT_MAX ? r : INFINITY));  // NaN too
}

// The screening table of a FLAT_SQ16 index: its stored rows as one exact fp16 plane, no mean, scale 1,
// the column term |x|^2 (L2) or 0 (IP); synchronises.  Only max |x|^2 is computed, for the tolerance.
static void tc_install_rows(dfx_index* idx, cudaStream_t st) {
    const int d = idx->cfg.d;
    const int64_t N = idx->n_sorted;
    dfx_tc_table& tab = idx->tc_tab;
    tab.mean.reserve((size_t)d * 4 + 8);  // m = 0, then the maximum
    float* max2 = tab.mean.as<float>() + d;
    DFX_CUDA(cudaMemsetAsync(tab.mean.p, 0, (size_t)d * 4 + 8, st));
    DFX_LAUNCH(rows_max2_kernel, (unsigned)dfx_ceil_div(N, 8), 256, 0, st, idx->payload.as<__half>(), N, d, max2);
    float h = 0.f;
    DFX_CUDA(cudaMemcpyAsync(&h, max2, 4, cudaMemcpyDeviceToHost, st));
    DFX_CUDA(cudaStreamSynchronize(st));
    tab.cmax2 = tab.cmax2c = h;
    tab.scale = 1.f;
    idx->tc_flat_finite = std::isfinite(h);
    if (idx->tc_mode == 0) idx->tc_fast = false;
    idx->tc_stat_pending = false;
    idx->tc_acc_rows = idx->tc_acc_bad = 0;
}

bool dfx_tc_flat_table(dfx_index* idx, cudaStream_t st) {
    const int64_t N = idx->n_sorted;
    const bool sq16 = idx->cfg.kind == DFX_FLAT_SQ16;
    if (idx->tc_flat_rows != N) {  // (re)build the screening table of the rows
        if (sq16) tc_install_rows(idx, st);
        else tc_install_table(idx, idx->payload.as<float>(), N, st);
        idx->tc_flat_rows = N;
    }
    if (sq16) {  // the rows may have moved (an add grows the store)
        idx->tc_tab.rows = idx->payload.as<__half>();
        idx->tc_tab.rows_cterm = idx->cfg.metric == DFX_METRIC_L2 ? idx->xnorm.as<float>() : nullptr;
    }
    return idx->tc_flat_finite;
}

int dfx_tc_flat_candidates(dfx_index* idx, const float* d_x, int64_t nq, int k, cudaStream_t st) {
    DFX_REQUIRE(dfx_tc_flat_covers(idx, k), "flat search on tensor cores: the shape is not covered");
    const int64_t N = idx->n_sorted;
    DFX_REQUIRE(idx->tc_flat_rows == N && idx->tc_flat_finite,
                "flat search on tensor cores: no usable screening table (dfx_tc_flat_table)");
    const int d = idx->cfg.d;
    const int metric = idx->cfg.metric;
    const int64_t nl_pad = dfx_ceil_div(N, tc::TILE) * tc::TILE;
    const int ng = (int)(nl_pad / 32);
    tc_stats_poll(idx, st);
    const bool fast = idx->tc_fast;
    int G = k + 8;
    if (G > ng) G = ng;
    const int ncand = G * 32;
    idx->tc_cand.reserve((size_t)nq * ncand * 8);
    const Screened s = tc_screen_chunk(idx, d, d_x, nq, nq, ng, G, idx->tc_tab, fast ? 1 : 2, N, metric, st);
    const ScreenTol tol = tc_tol(idx, idx->tc_tab, d, fast);
    dfx_with_flat_rows(idx, [&](auto rows) {
        using T = std::remove_cv_t<std::remove_pointer_t<decltype(rows)>>;
        auto kern = rerank_kernel<0, T>;
        DFX_LAUNCH(kern, (unsigned)nq, 128, (size_t)d * 4, st, d_x, d, rows, idx->xnorm.as<float>(), N, metric,
                   s.groups, G, k, s.gmin, s.gmin2, s.gargc, ng, tol, idx->tc_cand.as<uint64_t>(), (int32_t*)nullptr,
                   (const int32_t*)nullptr, (const int32_t*)nullptr, nq, (int32_t*)nullptr, s.ovf);
        // rows with more near-ties than selected groups: their ncand slots become the exact top-ncand
        launch_exact_rows(d_x, rows, idx->xnorm.as<float>(), N, d, metric, s.ovf, nq, 0, ncand, nullptr, nullptr,
                          idx->tc_cand.as<uint64_t>(), st);
    });
    tc_stats_post(idx, s.ovf, nq, fast, st);
    return ncand;
}

// nearest centroid per row (build path): screening, then the answer straight from the screening
// summary when it is unambiguous, exact canonical evaluation for the (rare) ambiguous rows
void dfx_tc_assign(dfx_index* idx, int d, const float* d_cent, const float* d_cnorm, int64_t nlist, int metric,
                   int64_t n, const float* d_x, int32_t* d_assign, cudaStream_t st) {
    const int64_t nl_pad = dfx_ceil_div(nlist, tc::TILE) * tc::TILE;
    const int ng = (int)(nl_pad / 32);
    // groups kept per row: the best one decides, the others tell whether it does so unambiguously;
    // a row whose G-th group is still within the tolerance goes to the exact fallback
    const int G = ng < 6 ? ng : 6;
    const int64_t RC = std::max<int64_t>(tc::TILE, ((256ll << 20) / ((int64_t)ng * 4)) / tc::TILE * tc::TILE);
    const int64_t rmax = std::min<int64_t>(n, RC);
    idx->tc_amb.reserve((size_t)(rmax + 1) * 4);
    // fp16 copy of this centroid table (k-means changes it every iteration; converting is cheap).
    // Precision: tc_mode 1 / 2 as set; AUTO decides per chunk from the counts of the chunk before
    // (read back with a sync -- this is the build path), starting PRECISE on every call.
    tc_prepare_table(d_cent, nlist, d, metric, idx->tc_tab_tmp, st);
    bool fast = idx->tc_mode == 1;
    int64_t acc_rows = 0, acc_bad = 0;
    for (int64_t r0 = 0, rc = 0; r0 < n; r0 += rc) {
        // the first AUTO chunk is a small PRECISE probe (16 384 rows), so that most of the rows run
        // at the precision their statistics call for
        rc = (idx->tc_mode == 0 && r0 == 0) ? std::min<int64_t>(n, dfx_ceil_div(idx->tc_auto_window, tc::TILE) * tc::TILE)
                                            : std::min(RC, n - r0);
        const float* xr = d_x + r0 * d;
        const Screened s = tc_screen_chunk(idx, d, xr, rc, rmax, ng, G, idx->tc_tab_tmp, fast ? 1 : 2, nlist, metric, st);
        const ScreenTol tol = tc_tol(idx, idx->tc_tab_tmp, d, fast);
        ScreenTol tol_rr = tol;
        tol_rr.rel_fast = 0.f;  // counted once per row by assign_resolve_kernel
        int32_t* amb_count = idx->tc_amb.as<int32_t>();
        int32_t* amb_rows = amb_count + 1;
        DFX_CUDA(cudaMemsetAsync(amb_count, 0, 4, st));
        DFX_LAUNCH(assign_resolve_kernel, (unsigned)dfx_ceil_div(rc, 256), 256, 0, st, s.groups, s.gmin, s.gmin2,
                   s.gargc, ng, G, tol, rc, d_assign + r0, amb_rows, amb_count, s.ovf);
        auto kern = rerank_kernel<1>;
        const unsigned grid = (unsigned)std::min<int64_t>(rc, dfx_num_sms() * 16);
        DFX_LAUNCH(kern, grid, 128, (size_t)d * 4, st, xr, d, d_cent, d_cnorm, nlist, metric, s.groups, G, 1, s.gmin,
                   s.gmin2, s.gargc, ng, tol_rr, (uint64_t*)nullptr, d_assign + r0, (const int32_t*)amb_rows,
                   (const int32_t*)amb_count, rc, (int32_t*)nullptr, s.ovf);
        launch_exact_rows(xr, d_cent, d_cnorm, nlist, d, metric, s.ovf, rc, 1, 1, nullptr, d_assign + r0, nullptr, st);
        if (idx->tc_mode == 0 && r0 + rc < n) {  // AUTO: the next chunk's precision
            int32_t h[2] = {0, 0};
            DFX_CUDA(cudaMemcpyAsync(h, s.ovf, 8, cudaMemcpyDeviceToHost, st));
            DFX_CUDA(cudaStreamSynchronize(st));
            fast = tc_auto_step(fast, rc, h[0], h[1], idx->tc_auto_window, acc_rows, acc_bad);
        }
    }
}
