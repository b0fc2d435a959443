// dfx_scan_pq4_dev.cuh -- K4 for 4-bit PQ codes (included by dfx_search.cu; also compiled by the
// CPU emulator, tests/emu/).
//
// Replaces the inner loop of faiss IndexIVFPQ::search for shards built with nbits = 4 (reference
// index.py:43-48 with bits_per_vector = 4):
//   v = dis0 + (t + S),  S = halving-tree sum over P = next_pow2(M) of lut[m][code_m] (oracle
//   pq_sum, positions m >= M hold +0).
// One CTA per (query, group of G consecutive probes) and one lane per vector, like scan_pq_kernel;
// the codes are the packed row-major rows (M / 2 bytes, code m in nibble m & 1 of byte m >> 1).
//
//   * The table lives in registers, not in shared memory.  A sub-table of 16 floats is half a
//     warp: lane L keeps T[j] = lut[2j + (L >> 4)][L & 15] for j < M / 2, so one SHFL from lane
//     ((m & 1) << 4) | code_m returns lut[m][code_m].  Every register index is a compile-time
//     constant (MT = M is a template argument), and a shuffle has no bank conflicts.  The table is
//     the global [queries][M][16] one of pq_prep_kernel; T[j] = lut[q][32 j + L] is one coalesced
//     load per register.
//   * The shuffles need all 32 lanes: lanes past the end of a list read the codes, t-value and id of
//     the warp's first row (a valid one), run the same lookups and are dropped at admission only.
//   * Registers: the tree's first level adds positions m and m + P / 2 while the codes are read
//     (a literal +0.f where m + P / 2 >= M, as the oracle's padding), so a lane keeps P / 2 partials;
//     dfx_halving_tree finishes the canonical order.
//   * Nibble extraction: the low and high nibbles of a code word are split once per word with the
//     lane-half bit already set (lo = w & 0x0f0f0f0f, hi = (w >> 4) & 0x0f0f0f0f | 0x10101010); SHFL
//     reads only the 5 low bits of its lane operand, so code m is then lo >> 8 b or hi >> 8 b.
#pragma once
#include "dfx_common.cuh"
#include "dfx_topk.cuh"

constexpr int PQ4_KSUB = 16;

// shared memory of one CTA: 4 per-warp candidate buffers of `cap` composites (MAT: none)
static inline size_t dfx_pq4_smem(int cap) { return (size_t)4 * cap * 8; }

// M = 40, 72, 88: under ptxas's default register budget one value is reloaded from local memory in
// the per-vector loop; asking for one resident block lets it keep everything in registers.  The other
// shapes keep the default (0), which spills only outside that loop and leaves more blocks per SM.
// MAT (k > 1024): `part` is the candidate buffer; every vector's composite goes to slot
// coff[q][p] + (position in list) (dfx_cand_store) instead of the per-warp queues.
template <int MT, bool MAT = false>
__global__ void __launch_bounds__(128, (MT == 40 || MT == 72 || MT == 88) ? 1 : 0)
scan_pq4_kernel(const float* __restrict__ lut, const float* __restrict__ dis0, const int32_t* __restrict__ keys,
                int nprobe, int G, int ngroups, const int64_t* __restrict__ list_off,
                const uint8_t* __restrict__ codes, const float* __restrict__ tvals, const int32_t* __restrict__ ids,
                int k, int cap, uint64_t* __restrict__ part, const int64_t* __restrict__ coff) {
    static_assert(MT >= 8 && MT <= 128 && MT % 8 == 0, "4-bit codes: M % 8 == 0, 8 <= M <= 128");
    constexpr int NW = MT / 8;  // 32-bit code words per row
    constexpr int P = (MT <= 8) ? 8 : (MT <= 16) ? 16 : (MT <= 32) ? 32 : (MT <= 64) ? 64 : 128;
    constexpr int H = P / 2;
    DFX_DYN_SMEM(unsigned char, smem_raw, 16);
    uint64_t* s_buf = reinterpret_cast<uint64_t*>(smem_raw);
    const int64_t q = blockIdx.x / ngroups;
    const int g = blockIdx.x % ngroups;
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;

    float T[MT / 2];
    {
        const float* lq = lut + q * (int64_t)MT * PQ4_KSUB;
#pragma unroll
        for (int j = 0; j < MT / 2; j++) T[j] = __ldg(lq + 32 * j + lane);
    }
    WarpTopK wt;
    if constexpr (!MAT) wt.init(s_buf + (size_t)warp * cap, cap, k);

    const int p_end = min(nprobe, (g + 1) * G);
    for (int p = g * G; p < p_end; p++) {
        const int l = keys[q * nprobe + p];
        if (l < 0) continue;
        const float d0 = dis0[q * nprobe + p];
        const int64_t beg = list_off[l], end = list_off[l + 1];
        int64_t cbase = 0;  // MAT: slot of row i is cbase + i
        if constexpr (MAT) cbase = coff[q * (nprobe + 1) + p] - beg;
        for (int64_t base = beg + warp * 32; base < end; base += 128) {  // warp-uniform trip count
            const int64_t i = base + lane;
            const bool valid = i < end;
            const int64_t r = valid ? i : base;  // tail lanes: the warp's first row
            uint32_t w[NW];
            if constexpr (NW % 4 == 0) {
                const uint4* cp = reinterpret_cast<const uint4*>(codes + r * (MT / 2));
#pragma unroll
                for (int c = 0; c < NW / 4; c++) {
                    const uint4 v4 = __ldg(cp + c);
                    w[4 * c + 0] = v4.x;
                    w[4 * c + 1] = v4.y;
                    w[4 * c + 2] = v4.z;
                    w[4 * c + 3] = v4.w;
                }
            } else if constexpr (NW % 2 == 0) {
                const uint2* cp = reinterpret_cast<const uint2*>(codes + r * (MT / 2));
#pragma unroll
                for (int c = 0; c < NW / 2; c++) {
                    const uint2 v2 = __ldg(cp + c);
                    w[2 * c + 0] = v2.x;
                    w[2 * c + 1] = v2.y;
                }
            } else {
                const uint32_t* cp = reinterpret_cast<const uint32_t*>(codes + r * (MT / 2));
#pragma unroll
                for (int c = 0; c < NW; c++) w[c] = __ldg(cp + c);
            }
            const uint32_t my_id = (uint32_t)__ldg(ids + r);  // loaded with the codes: no dependent load on admission
            const float t = __ldg(tvals + r);
            // lane operand of sub-quantizer m: word m >> 3, byte (m >> 1) & 3, nibble m & 1
            uint32_t lo[NW], hi[NW];
#pragma unroll
            for (int c = 0; c < NW; c++) {
                lo[c] = w[c] & 0x0f0f0f0fu;
                hi[c] = ((w[c] >> 4) & 0x0f0f0f0fu) | 0x10101010u;
            }
            auto look = [&](int m) {
                const uint32_t src = ((m & 1) ? hi[m >> 3] : lo[m >> 3]) >> (8 * ((m >> 1) & 3));
                return __shfl_sync(0xffffffffu, T[m >> 1], (int)src);
            };
            float s[H];
#pragma unroll
            for (int m = 0; m < H; m++) {
                const float a = look(m);
                if (m + H < MT) s[m] = a + look(m + H);
                else s[m] = a + 0.f;
            }
            if constexpr (H > 1) dfx_halving_tree<H / 2>(s);
            const float v = d0 + (t + s[0]);
            if constexpr (MAT) {
                if (valid) dfx_cand_store(part, cbase + i, v, my_id);
            } else {
                uint32_t sec = 0;
                const bool want = valid && wt.admits(v, [&] { return my_id; }, sec);
                wt.push_lanes(want, v, sec);
            }
        }
    }
    if constexpr (!MAT) cta_merge_and_write<128>(wt, s_buf, cap, k, part + ((int64_t)q * ngroups + g) * k);
}
