// dfx_scan_pq4_dev.cuh -- K4 for 4-bit PQ codes (included by dfx_search.cu; also compiled by the
// CPU emulator, tests/emu/).
//
// Replaces the inner loop of faiss IndexIVFPQ::search for shards built with nbits = 4 (reference
// index.py:43-48 with bits_per_vector = 4):
//   v = dis0 + (t + S),  S = halving-tree sum over P = next_pow2(M) of lut[m][code_m] (oracle
//   pq_sum, positions m >= M hold +0).
// The probe loop, the lane-per-vector walk and the candidate sink are the shared list-scan skeleton
// (dfx_scan_dev.cuh); the codes are the packed row-major rows (M / 2 bytes, code m in nibble m & 1 of byte m >> 1).
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
#include "dfx_scan_dev.cuh"

constexpr int PQ4_KSUB = 16;

// M = 40, 72, 88: under ptxas's default register budget one value is reloaded from local memory in
// the per-vector loop; asking for one resident block lets it keep everything in registers.  The other
// shapes keep the default (0), which spills only outside that loop and leaves more blocks per SM.
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
    const ScanProbes pr(keys, dis0, list_off, nprobe, G, ngroups);
    const int lane = threadIdx.x & 31;

    float T[MT / 2];
    {
        const float* lq = lut + pr.q * (int64_t)MT * PQ4_KSUB;
#pragma unroll
        for (int j = 0; j < MT / 2; j++) T[j] = __ldg(lq + 32 * j + lane);
    }
    ScanSink<MAT, 128> sink(reinterpret_cast<uint64_t*>(smem_raw), cap, k, part, coff);

    dfx_scan_lanes<true>(pr, sink, [&](int64_t i, bool valid, int64_t base, float d0) {
        const int64_t r = valid ? i : base;  // tail lanes: the warp's first row
        uint32_t w[NW];
        dfx_load_code_words(codes + r * (MT / 2), w);
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
        return ScanCand{d0 + (t + s[0]), my_id};
    });
    sink.finish(pr);
}
