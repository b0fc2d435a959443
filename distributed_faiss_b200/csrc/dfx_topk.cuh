// dfx_topk.cuh -- per-warp / per-CTA k-selection used by the inverted-list scan kernels.
#pragma once
#include "dfx_common.cuh"
#include "dfx_select.cuh"

// ascending bitonic sort of buf[0, cnt) by one warp: the slots up to P = the next power of two
// >= max(cnt, 32) are padded with NONE and sorted with them; returns P
__device__ __forceinline__ int dfx_warp_sort_buf(uint64_t* buf, int cnt, int lane) {
    int P = 32;
    while (P < cnt) P <<= 1;
    for (int e = cnt + lane; e < P; e += 32) buf[e] = DFX_COMP_NONE;
    __syncwarp();
    for (int size = 2; size <= P; size <<= 1) {
        for (int stride = size >> 1; stride > 0; stride >>= 1) {
            for (int i = lane; i < (P >> 1); i += 32) {
                const int pos = 2 * i - (i & (stride - 1));
                const int partner = pos + stride;
                const bool up = ((pos & size) == 0);
                const uint64_t a = buf[pos], b = buf[partner];
                if ((a > b) == up) {
                    buf[pos] = b;
                    buf[partner] = a;
                }
            }
            __syncwarp();
        }
    }
    return P;
}

// =====================================================================================
// per-warp candidate set: keeps the k best composites seen so far in shared memory.
// buf has CAP = 2*KP slots (KP = pow2 >= max(k,32)); when it cannot take another 32
// entries it is bitonic-sorted by the warp and cut back to k; thr = current k-th value.
// =====================================================================================
struct WarpTopK {
    uint64_t* buf;
    int cap, k, cnt;
    float thr;         // value of the current k-th best (+inf until k candidates are held)
    uint32_t thr_sec;  // its secondary key: an equal value is only admitted with a smaller one
    // optional CTA-wide bound: the smallest k-th-best value any warp of the CTA has reached so
    // far (monotone uint key in shared memory).  Every warp's k-th best is an upper bound of the
    // CTA's k-th best, so a candidate above it can never be in the CTA's result; candidates equal
    // to it are still admitted (their rank is decided by the id at merge time).
    unsigned int* cta_key = nullptr;
    __device__ __forceinline__ void init(uint64_t* b, int cap_, int k_, unsigned int* cta_key_ = nullptr) {
        buf = b;
        cap = cap_;
        k = k_;
        cnt = 0;
        thr = __int_as_float(0x7f800000);  // +inf
        thr_sec = DFX_SEC_NONE;
        cta_key = cta_key_;
    }
    // current CTA-wide bound as a float (call once per block of work, it is one broadcast LDS)
    __device__ __forceinline__ float cta_bound() const {
        return cta_key ? dfx_key2f(*reinterpret_cast<volatile unsigned int*>(cta_key)) : __int_as_float(0x7f800000);
    }
    // does (v, sec) beat the current k-th best?  `sec` is fetched lazily: only on a value tie
    template <class SecFn>
    __device__ __forceinline__ bool admits(float v, SecFn sec_of, uint32_t& sec) const {
        v = v + 0.0f;
        if (v < thr) {
            sec = sec_of();
            return true;
        }
        if (v == thr) {
            sec = sec_of();
            return sec < thr_sec;
        }
        return false;
    }
    __device__ __forceinline__ void sort_and_cut() {
        const int lane = threadIdx.x & 31;
        // sort only as many slots as are live; slots beyond P are never read before they are
        // overwritten by later pushes
        dfx_warp_sort_buf(buf, cnt, lane);
        if (cnt > k) cnt = k;
        if (cnt == k) {
            const uint64_t kth = buf[k - 1];
            thr = dfx_key2f((uint32_t)(kth >> 32));
            thr_sec = (uint32_t)kth;
            if (cta_key && (threadIdx.x & 31) == 0) atomicMin(cta_key, (unsigned int)(kth >> 32));
        }
        __syncwarp();
    }
    // each lane may contribute one candidate (want = lane has one)
    __device__ __forceinline__ void push_lanes(bool want, float v, uint32_t sec) {
        unsigned mask = __ballot_sync(0xffffffffu, want);
        if (mask == 0) return;
        const int lane = threadIdx.x & 31;
        if (want) buf[cnt + __popc(mask & ((1u << lane) - 1u))] = dfx_comp(v, sec);
        cnt += __popc(mask);
        __syncwarp();
        if (cnt > cap - 32) sort_and_cut();
    }
    // warp-uniform single candidate
    __device__ __forceinline__ void push_uniform(float v, uint32_t sec) {
        if ((threadIdx.x & 31) == 0) buf[cnt] = dfx_comp(v, sec);
        cnt += 1;
        __syncwarp();
        if (cnt > cap - 32) sort_and_cut();
    }
};

// The other sink of the list scans (MAT = true, searches with k > 1024): the composite of every
// scanned vector goes to its own slot of the query's candidate row, and one k-selection per query
// picks the result (dfx_search.cu).  WarpTopK::admits never takes a NaN value; it is stored as "none".
__device__ __forceinline__ void dfx_cand_store(uint64_t* cand, int64_t pos, float v, uint32_t id) {
    cand[pos] = (v == v) ? dfx_comp(v, id) : DFX_COMP_NONE;
}

// merges the per-warp sets of a CTA and writes k composites (NONE padded) to out.
// Each warp first sorts and cuts its own set to <= k entries; only those live entries
// (NW*k of the NW*cap slots) are then packed densely and sorted by the CTA.
template <int THREADS>
__device__ __forceinline__ void cta_merge_and_write(WarpTopK& wt, uint64_t* s_buf, int cap, int k,
                                                    uint64_t* out) {
    wt.sort_and_cut();
    constexpr int NW = THREADS / 32;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (k <= 128) {
        uint64_t mine[4];
#pragma unroll
        for (int i = 0; i < 4; i++) {
            const int j = lane + 32 * i;
            mine[i] = (j < wt.cnt) ? wt.buf[j] : DFX_COMP_NONE;
        }
        __syncthreads();  // every warp has its live entries in registers: s_buf can be reused
#pragma unroll
        for (int i = 0; i < 4; i++) {
            const int j = lane + 32 * i;
            if (j < k) s_buf[warp * k + j] = mine[i];
        }
        int P = 32;
        while (P < NW * k) P <<= 1;
        for (int e = NW * k + threadIdx.x; e < P; e += THREADS) s_buf[e] = DFX_COMP_NONE;
        dfx_block_bitonic_sort<THREADS>(s_buf, P);
    } else {
        // full-width path: everything beyond each warp's live entries must read as "none"
        for (int e = wt.cnt + lane; e < cap; e += 32) wt.buf[e] = DFX_COMP_NONE;
        __syncthreads();
        dfx_block_bitonic_sort<THREADS>(s_buf, NW * cap);
    }
    for (int j = threadIdx.x; j < k; j += THREADS) out[j] = s_buf[j];
}

// =====================================================================================
// register-resident variants: one 64-bit composite per lane, bitonic networks over shuffles
// =====================================================================================
// ascending bitonic sort of one 64-bit value per lane
__device__ __forceinline__ uint64_t dfx_warp_sort32_asc(uint64_t x, int lane) {
#pragma unroll
    for (int size = 2; size <= 32; size <<= 1) {
#pragma unroll
        for (int stride = size >> 1; stride >= 1; stride >>= 1) {
            const uint64_t o = __shfl_xor_sync(0xffffffffu, x, stride);
            const bool up = (lane & size) == 0;  // size == 32: true for every lane
            const bool lower = (lane & stride) == 0;
            const uint64_t mn = x < o ? x : o, mx = x < o ? o : x;
            x = (lower == up) ? mn : mx;
        }
    }
    return x;
}
// kept, x_asc: ascending over lanes.  returns the 32 smallest of their union, ascending.
// (element-wise min of an ascending and a descending sequence is bitonic and holds the 32
// smallest; five half-cleaner stages sort it)
__device__ __forceinline__ uint64_t dfx_warp_merge_sorted32(uint64_t kept, uint64_t x_asc, int lane) {
    const uint64_t xr = __shfl_sync(0xffffffffu, x_asc, 31 - lane);
    uint64_t y = kept < xr ? kept : xr;
#pragma unroll
    for (int stride = 16; stride >= 1; stride >>= 1) {
        const uint64_t o = __shfl_xor_sync(0xffffffffu, y, stride);
        const bool lower = (lane & stride) == 0;
        const uint64_t mn = y < o ? y : o, mx = y < o ? o : y;
        y = lower ? mn : mx;
    }
    return y;
}
