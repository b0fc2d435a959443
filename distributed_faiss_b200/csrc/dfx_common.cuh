// dfx_common.cuh -- shared device/host helpers for libdfx (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <cuda_fp16.h>
#include <stdint.h>
#include <float.h>
#include <string>
#include <atomic>

#include "../../include/dfx.h"

// IVF-SQ8 decode (faiss QT_8bit, DESIGN.md section 2): t = fmaf(code, SCALE, BIAS)
constexpr float DFX_SQ8_SCALE = 1.f / 255.f;
constexpr float DFX_SQ8_BIAS = 0.5f / 255.f;

// ---------------------------------------------------------------- errors
void dfx_set_error(const std::string& msg);
extern std::atomic<long long> g_dfx_launches;

struct DfxError {
    std::string msg;
};

#define DFX_CUDA(expr)                                                                       \
    do {                                                                                     \
        cudaError_t _e = (expr);                                                             \
        if (_e != cudaSuccess) {                                                             \
            throw DfxError{std::string(#expr) + " failed: " + cudaGetErrorString(_e) + " (" + \
                           __FILE__ + ":" + std::to_string(__LINE__) + ")"};                 \
        }                                                                                    \
    } while (0)

#define DFX_REQUIRE(cond, msg)                  \
    do {                                        \
        if (!(cond)) throw DfxError{(msg)};     \
    } while (0)

// every kernel launch goes through this so that dfx_launch_count() is honest
#ifdef DFX_EMU
// CPU emulator build (tests/emu/, never a product build): the kernel runs on the fiber SIMT
// runtime, one CTA after the other, synchronously.  Every launch is recorded so that tests can
// tell which instantiation a search ran (tests/emu/emu_simt_impl.cpp, dfx_emu_launch_log).  The
// recorder is weak: an emulator build whose runtime does not define it records nothing.
__attribute__((weak)) void dfx_emu_record_launch(const void* kernel);
#define DFX_LAUNCH(kernel, grid, block, smem, stream, ...)                                      \
    do {                                                                                        \
        const dim3 _g(grid), _b(block);                                                         \
        const auto _kfn = kernel;                                                               \
        if (dfx_emu_record_launch) dfx_emu_record_launch(reinterpret_cast<const void*>(_kfn));  \
        simt::launch3(_g.x, _g.y, _b.x, (size_t)(smem), [&]() { kernel(__VA_ARGS__); });         \
        g_dfx_launches.fetch_add(1, std::memory_order_relaxed);                                 \
    } while (0)
#else
#define DFX_LAUNCH(kernel, grid, block, smem, stream, ...)                                      \
    do {                                                                                        \
        const dim3 _g(grid), _b(block);                                                         \
        kernel<<<_g, _b, (smem), (stream)>>>(__VA_ARGS__);                                      \
        g_dfx_launches.fetch_add(1, std::memory_order_relaxed);                                 \
        cudaError_t _le = cudaGetLastError();                                                   \
        if (_le != cudaSuccess)                                                                 \
            throw DfxError{std::string("launch of " #kernel " failed: ") + cudaGetErrorString(_le) + \
                           " grid=(" + std::to_string(_g.x) + "," + std::to_string(_g.y) + ") block=" + \
                           std::to_string(_b.x) + " smem=" + std::to_string((size_t)(smem)) + " (" +  \
                           __FILE__ + ":" + std::to_string(__LINE__) + ")"};                    \
    } while (0)
#endif

// grow-only device buffer
struct DevBuf {
    void* p = nullptr;
    size_t cap = 0;
    DevBuf() = default;
    DevBuf(const DevBuf&) = delete;
    DevBuf& operator=(const DevBuf&) = delete;
    DevBuf(DevBuf&& o) noexcept : p(o.p), cap(o.cap) {
        o.p = nullptr;
        o.cap = 0;
    }
    DevBuf& operator=(DevBuf&& o) noexcept {
        if (this != &o) {
            release();
            p = o.p;
            cap = o.cap;
            o.p = nullptr;
            o.cap = 0;
        }
        return *this;
    }
    ~DevBuf() { release(); }
    void release() {
        if (p) cudaFree(p);
        p = nullptr;
        cap = 0;
    }
    // ensure capacity; contents are NOT preserved unless keep_bytes > 0
    void reserve(size_t bytes, size_t keep_bytes = 0, cudaStream_t st = 0) {
        if (bytes <= cap) return;
        void* np_ = nullptr;
        DFX_CUDA(cudaMalloc(&np_, bytes));
        if (p && keep_bytes) {
            DFX_CUDA(cudaMemcpyAsync(np_, p, keep_bytes, cudaMemcpyDeviceToDevice, st));
            DFX_CUDA(cudaStreamSynchronize(st));
        }
        if (p) cudaFree(p);
        p = np_;
        cap = bytes;
    }
    template <typename T>
    T* as() const {
        return reinterpret_cast<T*>(p);
    }
};

// ---------------------------------------------------------------- ordering keys
// Everything on device minimises a float "value" (distance, or -inner_product) and breaks
// ties on a 32-bit secondary key (local id / column / position): composite = key<<32 | sec.
#define DFX_SEC_NONE 0xffffffffu
#define DFX_COMP_NONE 0xffffffffffffffffull

__host__ __device__ __forceinline__ uint32_t dfx_f2key(float v) {
    v = v + 0.0f;  // -0.0 -> +0.0 so that equal floats give equal keys
#ifdef __CUDA_ARCH__
    uint32_t u = __float_as_uint(v);
#else
    uint32_t u;
    memcpy(&u, &v, 4);
#endif
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__host__ __device__ __forceinline__ float dfx_key2f(uint32_t k) {
    uint32_t u = (k & 0x80000000u) ? (k & 0x7fffffffu) : ~k;
#ifdef __CUDA_ARCH__
    return __uint_as_float(u);
#else
    float f;
    memcpy(&f, &u, 4);
    return f;
#endif
}
__device__ __forceinline__ uint64_t dfx_comp(float v, uint32_t sec) {
    return ((uint64_t)dfx_f2key(v) << 32) | (uint64_t)sec;
}

// ---------------------------------------------------------------- canonical arithmetic (device)
// halving tree of the PQ sums: v[r] += v[r + OFF] for OFF, OFF / 2, ..., 1; the sum lands in v[0].
// (recursion, not a loop over OFF: ptxas for sm_90a keeps a loop-carried halving step in local memory)
template <int OFF, int N>
__device__ __forceinline__ void dfx_halving_tree(float (&v)[N]) {
    static_assert(2 * OFF <= N, "tree wider than the array");
#pragma unroll
    for (int r = 0; r < OFF; r++) v[r] = v[r] + v[r + OFF];
    if constexpr (OFF > 1) dfx_halving_tree<OFF / 2>(v);
}
// warp-dot: lane j owns k = 128*i + 4*j + t; butterfly xor 16,8,4,2,1 (DESIGN.md)
__device__ __forceinline__ float dfx_warp_butterfly(float acc) {
#pragma unroll
    for (int off = 16; off >= 1; off >>= 1) acc = acc + __shfl_xor_sync(0xffffffffu, acc, off);
    return acc;
}
// seq-k dot product q . x: acc = fma(q[k], x[k], acc), k ascending (oracle/dfx_oracle.c).
// d % 4 == 0 and x 16-byte aligned: float4 row loads, unrolled so that 8 are in flight.
__device__ __forceinline__ float dfx_dot_seqk(const float* q, const float* x, int d) {
    float acc = 0.f;
#pragma unroll 8
    for (int k = 0; k < d; k += 4) {
        const float4 xv = *reinterpret_cast<const float4*>(x + k);
        acc = __fmaf_rn(q[k + 0], xv.x, acc);
        acc = __fmaf_rn(q[k + 1], xv.y, acc);
        acc = __fmaf_rn(q[k + 2], xv.z, acc);
        acc = __fmaf_rn(q[k + 3], xv.w, acc);
    }
    return acc;
}
// the same over fp16 rows (FLAT_SQ16): each element widened exactly, the same chain of fmas, so the
// value equals the one over the fp32 rows they decode to.  d % 4 == 0, x 8-byte aligned.
__device__ __forceinline__ float dfx_dot_seqk(const float* q, const __half* x, int d) {
    float acc = 0.f;
#pragma unroll 8
    for (int k = 0; k < d; k += 4) {
        const __half2* xh = reinterpret_cast<const __half2*>(x + k);
        const float2 a = __half22float2(xh[0]), b = __half22float2(xh[1]);
        acc = __fmaf_rn(q[k + 0], a.x, acc);
        acc = __fmaf_rn(q[k + 1], a.y, acc);
        acc = __fmaf_rn(q[k + 2], b.x, acc);
        acc = __fmaf_rn(q[k + 3], b.y, acc);
    }
    return acc;
}
// one stored element as fp32 (exact for both row types)
__device__ __forceinline__ float dfx_elem_f32(float v) { return v; }
__device__ __forceinline__ float dfx_elem_f32(__half v) { return __half2float(v); }
// ranking value of column col from its inner product with the query: -ip (IP), or |x|^2 - 2 ip
// (L2, |q|^2 left out); xnorm is only read for L2
__device__ __forceinline__ float dfx_rank_value(float ip, int metric, const float* xnorm, int64_t col) {
    return (metric == DFX_METRIC_IP) ? -ip : __fmaf_rn(-2.f, ip, xnorm[col]);
}

// IEEE division, round to nearest (spelled out so that no compiler setting can relax it)
__device__ __forceinline__ float dfx_div_rn(float a, float b) {
#ifdef DFX_EMU
    return a / b;
#else
    return __fdiv_rn(a, b);
#endif
}

// code of sub-quantizer m of row i of IVF-PQ codes stored with NB bits per code: NB = 8, one byte
// per code (u8[n][M]); NB = 4, packed as faiss does (u8[n][M / 2], code m in nibble m & 1 of byte
// m >> 1, low nibble first)
template <int NB>
__device__ __forceinline__ int dfx_pq_code(const uint8_t* codes, int64_t i, int M, int m) {
    static_assert(NB == 8 || NB == 4, "4 or 8 bits per code");
    if constexpr (NB == 4) return (codes[i * (M / 2) + (m >> 1)] >> ((m & 1) * 4)) & 15;
    else return codes[i * M + m];
}

// the list l with off[l] <= key < off[l + 1] (binary search over off[0..nlist]): the list that holds
// position key of list-sorted storage (off = list_off), or block key of the interleaved storage
// (off = blk_off)
__device__ __forceinline__ int64_t dfx_list_of(const int64_t* __restrict__ off, int64_t nlist, int64_t key) {
    int64_t lo = 0, hi = nlist;
    while (hi - lo > 1) {
        int64_t mid = (lo + hi) >> 1;
        if (off[mid] <= key) lo = mid; else hi = mid;
    }
    return lo;
}

static inline int64_t dfx_ceil_div(int64_t a, int64_t b) { return (a + b - 1) / b; }
static inline int dfx_next_pow2(int x) {
    int p = 1;
    while (p < x) p <<= 1;
    return p;
}
