// dfx_scan_dev.cuh -- the skeleton of every IVF list scan but scan_pq_il2_kernel: scan_rows_kernel
// and scan_pq_kernel (dfx_search.cu), scan_pq_wide_kernel, scan_pq4_kernel and scan_pq_fs_kernel, and
// their queue sizing (included by their files; also compiled by the CPU emulator, tests/emu/).
//
// One CTA scans the lists of one query's group of G consecutive probes (blockIdx.x = q * ngroups + g)
// and leaves the k best of them in the group's row of `part`.  A scan writes its table staging and
// its per-vector value; this header holds the rest:
//   ScanProbes           the CTA's (q, g) and the loop over its non-empty probes
//   ScanSink<MAT, T>     where the values go: per-warp WarpTopK queues, merged into the group's row at
//                        the end, or (MAT, k > 1024) each vector's composite in its own slot of the
//                        query's candidate row (dfx_search.cu, "k > 1024")
//   dfx_scan_lanes       the lane-per-vector walk of the PQ scans
//   dfx_load_code_words  a row's 32-bit code words in the widest loads its length allows
#pragma once
#include "dfx_common.cuh"
#include "dfx_topk.cuh"

// shared memory of the candidate queues of a `threads`-thread CTA: `cap` composites per warp, none
// when MAT
static inline size_t dfx_scan_queue_smem(int threads, int cap, bool mat) {
    return mat ? 0 : (size_t)(threads / 32) * cap * 8;
}

// the lists of the CTA's query q and probe group g: probes g * G .. min(nprobe, (g + 1) * G)
struct ScanProbes {
    const int32_t* keys;     // [q][p]: the probed lists, < 0 for none
    const float* dis0;       // [q][p]: |q - c|^2 of the probed list (the PQ scans)
    const int64_t* list_off;
    int nprobe, G, ngroups;
    int64_t q;
    int g;
    __device__ __forceinline__ ScanProbes(const int32_t* keys_, const float* dis0_, const int64_t* list_off_,
                                          int nprobe_, int G_, int ngroups_)
        : keys(keys_), dis0(dis0_), list_off(list_off_), nprobe(nprobe_), G(G_), ngroups(ngroups_),
          q(blockIdx.x / ngroups_), g(blockIdx.x % ngroups_) {}

    // for each non-empty probe p with list l: enter(l), the sink's slot base of the list, then
    // body(beg, end, d0) over the list's rows [beg, end).  d0 = dis0[q][p] when DIS0, else 0 (a
    // compile-time choice: a scan without dis0 does not test for it).
    template <bool DIS0, class Sink, class Enter, class Body>
    __device__ __forceinline__ void for_each_list(Sink& sink, Enter enter, Body body) const {
        const int p_end = min(nprobe, (g + 1) * G);
        for (int p = g * G; p < p_end; p++) {
            const int l = keys[q * nprobe + p];
            if (l < 0) continue;
            float d0 = 0.f;
            if constexpr (DIS0) d0 = dis0[q * nprobe + p];
            enter(l);
            const int64_t beg = list_off[l], end = list_off[l + 1];
            sink.enter_list(q, nprobe, p, beg);
            body(beg, end, d0);
        }
    }
};

// The values of a THREADS-thread CTA.  !MAT: each warp keeps its k best in a WarpTopK queue of `cap`
// composites (warp w's at s_buf + w * cap) and finish() merges them into the group's row of `part`.
// MAT: `part` is the candidate buffer and the composite of row i of probe p's list goes to slot
// coff[q][p] + (i - beg) (dfx_cand_store); no queues and no shared memory.
template <bool MAT, int THREADS>
struct ScanSink {
    WarpTopK wt;
    uint64_t* s_buf;
    uint64_t* part;
    const int64_t* coff;
    int64_t cbase = 0;  // MAT: slot of row i of the current list is cbase + i
    int cap, k;
    __device__ __forceinline__ ScanSink(uint64_t* s_buf_, int cap_, int k_, uint64_t* part_, const int64_t* coff_)
        : s_buf(s_buf_), part(part_), coff(coff_), cap(cap_), k(k_) {
        const int warp = (int)threadIdx.x >> 5;
        if constexpr (!MAT) wt.init(s_buf + (size_t)warp * cap, cap, k);
    }
    __device__ __forceinline__ void enter_list(int64_t q, int nprobe, int p, int64_t beg) {
        if constexpr (MAT) cbase = coff[q * (nprobe + 1) + p] - beg;
    }
    // one value per lane: row i, id `id`; lanes without a row (!valid) are dropped at admission.  The
    // id is only read by the queue on a value tie.
    __device__ __forceinline__ void push_lanes(bool valid, int64_t i, float v, uint32_t id) {
        if constexpr (MAT) {
            if (valid) dfx_cand_store(part, cbase + i, v, id);
        } else {
            uint32_t sec = 0;
            const bool want = valid && wt.admits(v, [&] { return id; }, sec);
            wt.push_lanes(want, v, sec);
        }
    }
    // one warp-uniform value for row i; under MAT lane `writer` stores it
    __device__ __forceinline__ void push_uniform(bool valid, int writer, int64_t i, float v, uint32_t id) {
        if constexpr (MAT) {
            if (((int)threadIdx.x & 31) == writer && valid) dfx_cand_store(part, cbase + i, v, id);
        } else {
            uint32_t sec = 0;
            if (valid && wt.admits(v, [&] { return id; }, sec)) wt.push_uniform(v, sec);
        }
    }
    __device__ __forceinline__ void finish(const ScanProbes& pr) {
        if constexpr (!MAT)
            cta_merge_and_write<THREADS>(wt, s_buf, cap, k, part + ((int64_t)pr.q * pr.ngroups + pr.g) * k);
    }
};

struct ScanCand {
    float v;
    uint32_t id;
};
// One lane per vector: warp w takes rows beg + 32 w + THREADS j of each list (a warp-uniform trip
// count).  value(i, valid, base, d0) returns the {value, id} of the lane's row i; valid = i < end,
// base = the warp's first row (always valid).  Tail lanes may compute on a row of their choice or not
// at all: the sink drops them.
template <bool DIS0, bool MAT, int THREADS, class Value>
__device__ __forceinline__ void dfx_scan_lanes(const ScanProbes& pr, ScanSink<MAT, THREADS>& sink, Value value) {
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    pr.for_each_list<DIS0>(sink, [](int) {}, [&](int64_t beg, int64_t end, float d0) {
        for (int64_t base = beg + warp * 32; base < end; base += THREADS) {
            const int64_t i = base + lane;
            const bool valid = i < end;
            const ScanCand c = value(i, valid, base, d0);
            sink.push_lanes(valid, i, c.v, c.id);
        }
    });
}

// the NW 32-bit code words of a row (16-byte aligned when NW % 4 == 0, 8-byte when NW % 2 == 0)
template <int NW>
__device__ __forceinline__ void dfx_load_code_words(const uint8_t* row, uint32_t (&w)[NW]) {
    if constexpr (NW % 4 == 0) {
        const uint4* cp = reinterpret_cast<const uint4*>(row);
#pragma unroll
        for (int c = 0; c < NW / 4; c++) {
            const uint4 v4 = __ldg(cp + c);
            w[4 * c + 0] = v4.x;
            w[4 * c + 1] = v4.y;
            w[4 * c + 2] = v4.z;
            w[4 * c + 3] = v4.w;
        }
    } else if constexpr (NW % 2 == 0) {
        const uint2* cp = reinterpret_cast<const uint2*>(row);
#pragma unroll
        for (int c = 0; c < NW / 2; c++) {
            const uint2 v2 = __ldg(cp + c);
            w[2 * c + 0] = v2.x;
            w[2 * c + 1] = v2.y;
        }
    } else {
        const uint32_t* cp = reinterpret_cast<const uint32_t*>(row);
#pragma unroll
        for (int c = 0; c < NW; c++) w[c] = __ldg(cp + c);
    }
}
