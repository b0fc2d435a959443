// dfx_build.cu -- building a shard on device: k-means (coarse centroids, PQ codebooks),
// assign + encode, and folding staged rows into contiguous inverted lists.
//
// Replaces `faiss_index.train(x)` (reference distributed_faiss/index.py:217) and
// `faiss_index.add(x)` (index.py:425).  Not on the timed search path (SURVEY.md 8f next-1),
// but required to produce a searchable shard without any CPU fallback.
// faiss semantics restated: Clustering = Lloyd iterations from a random subset, at most
// 256 points per centroid, empty clusters re-seeded from a large one; ProductQuantizer
// trained on residuals of <= 256*ksub training vectors; the 8-bit scalar quantizer on the
// per-dimension range of residuals of <= 100000 of them; add = nearest centroid under the
// quantizer's metric, ids sequential, ids ascending inside every list.
#include "dfx_internal.h"
#include "dfx_ptx.cuh"
#include <cub/cub.cuh>
#include <algorithm>
#include <numeric>
#include <random>

// ------------------------------------------------------------------ small kernels
__global__ void gather_rows_kernel(const float* __restrict__ src, const int32_t* __restrict__ rows,
                                   int64_t n, int d, int col0, int dsrc, float* __restrict__ dst) {
    int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= n * d) return;
    int64_t i = t / d;
    int c = (int)(t - i * d);
    int64_t r = rows ? rows[i] : i;
    dst[t] = src[r * dsrc + col0 + c];
}

__global__ void residual_kernel(const float* __restrict__ x, const float* __restrict__ cent,
                                const int32_t* __restrict__ assign, int64_t n, int d,
                                float* __restrict__ out) {
    int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= n * d) return;
    int64_t i = t / d;
    int c = (int)(t - i * d);
    out[t] = x[t] - cent[(size_t)assign[i] * d + c];
}

__global__ void count_kernel(const int32_t* __restrict__ keys, int64_t n, int32_t* __restrict__ cnt) {
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) atomicAdd(&cnt[keys[i]], 1);
}

__global__ void iota_kernel(int32_t* p, int64_t n) {
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) p[i] = (int32_t)i;
}

// one CTA per centroid: mean of its rows, rows visited in ascending row index (deterministic)
__global__ void centroid_update_kernel(const float* __restrict__ x, int d,
                                       const int32_t* __restrict__ order,
                                       const int32_t* __restrict__ seg_off,
                                       float* __restrict__ cent) {
    const int c = blockIdx.x;
    const int beg = seg_off[c], end = seg_off[c + 1];
    if (end <= beg) return;  // empty: keep the old centroid, handled by the host
    const float inv = 1.0f / (float)(end - beg);
    for (int k = threadIdx.x; k < d; k += blockDim.x) {
        float s = 0.f;
        for (int r = beg; r < end; r++) s += x[(size_t)order[r] * d + k];
        cent[(size_t)c * d + k] = s * inv;
    }
}

__global__ void split_cluster_kernel(float* cent, int d, int empty, int big) {
    int k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= d) return;
    const float eps = 1.f / 1024.f;
    float v = cent[(size_t)big * d + k];
    if ((k & 1) == 0) {
        cent[(size_t)empty * d + k] = v * (1 + eps);
        cent[(size_t)big * d + k] = v * (1 - eps);
    } else {
        cent[(size_t)empty * d + k] = v * (1 - eps);
        cent[(size_t)big * d + k] = v * (1 + eps);
    }
}

// PQ encode: grid (ceil(n/256), M); code_m = argmin_j l2_seq(r_m, P[m][j]), ties -> smaller j.
// The residual sub-vector lives in registers (DS = dsub when it is one of the common sizes).
// RES = false (IVF-PQ FastScan, not by_residual): r = x itself; cent and assign are not read.
template <int DS, bool RES = true>
__global__ void __launch_bounds__(256)
pq_encode_kernel(const float* __restrict__ x, const float* __restrict__ cent,
                 const int32_t* __restrict__ assign, int64_t n, int d, int M, int ksub, int dsub,
                 const float* __restrict__ codebooks, uint8_t* __restrict__ codes) {
    DFX_DYN_SMEM0(float, s_cb);  // [ksub][dsub]
    const int m = blockIdx.y;
    for (int i = threadIdx.x; i < ksub * dsub; i += blockDim.x)
        s_cb[i] = codebooks[(size_t)m * ksub * dsub + i];
    __syncthreads();
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float* xi = x + i * d + m * dsub;
    const float* c = RES ? cent + (size_t)assign[i] * d + m * dsub : nullptr;
    float best = FLT_MAX;
    int bj = 0;
    if (DS > 0) {
        float r[DS > 0 ? DS : 1];
#pragma unroll
        for (int t = 0; t < DS; t++) r[t] = RES ? xi[t] - c[t] : xi[t];
        for (int j = 0; j < ksub; j++) {
            float acc = 0.f;
#pragma unroll
            for (int t = 0; t < DS; t++) {
                float df = r[t] - s_cb[j * DS + t];
                acc = __fmaf_rn(df, df, acc);
            }
            if (acc < best) {
                best = acc;
                bj = j;
            }
        }
    } else {
        for (int j = 0; j < ksub; j++) {
            float acc = 0.f;
            for (int t = 0; t < dsub; t++) {
                float df = (RES ? xi[t] - c[t] : xi[t]) - s_cb[j * dsub + t];
                acc = __fmaf_rn(df, df, acc);
            }
            if (acc < best) {
                best = acc;
                bj = j;
            }
        }
    }
    codes[i * M + m] = (uint8_t)bj;
}

// IVF-PQR: the residual left after PQ1, r2 = (x - c) - P1[m][code_m], one fp32 rounding per
// subtraction.  cent == nullptr: x already holds the residuals x - c (training).
__global__ void pq_residual2_kernel(const float* __restrict__ x, const float* __restrict__ cent,
                                    const int32_t* __restrict__ assign, const uint8_t* __restrict__ codes, int64_t n,
                                    int d, int M, int dsub, const float* __restrict__ codebooks,
                                    float* __restrict__ out) {
    int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= n * d) return;
    int64_t i = t / d;
    int c = (int)(t - i * d);
    const int m = c / dsub;
    const float r1 = cent ? x[t] - cent[(size_t)assign[i] * d + c] : x[t];
    out[t] = r1 - codebooks[((size_t)m * 256 + codes[i * M + m]) * dsub + (c - m * dsub)];
}

// 4-bit codes: u8[n][M] (one code per byte, from pq_encode_kernel) -> the packed rows u8[n][M / 2].
// One thread per output byte, so no two threads write the same byte.
__global__ void pq_pack4_kernel(const uint8_t* __restrict__ in, int64_t nbytes, uint8_t* __restrict__ out) {
    int64_t b = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (b < nbytes) out[b] = (uint8_t)(in[2 * b] | (in[2 * b + 1] << 4));
}

// tvals[i] = sum_m ( |p_m|^2 + 2 <c_m, p_m> ), sequential in m (oracle orc_pq_tvals); NB = bits per
// stored code (dfx_pq_code)
template <int NB>
__global__ void pq_tvals_kernel(const uint8_t* __restrict__ codes, const int32_t* __restrict__ list_of,
                                const int64_t* __restrict__ list_off, int64_t nlist, int64_t n, int d,
                                int M, int ksub, int dsub, const float* __restrict__ codebooks,
                                const float* __restrict__ cent, float* __restrict__ tvals) {
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    int64_t l;
    if (list_of) l = list_of[i];
    else l = dfx_list_of(list_off, nlist, i);  // list-sorted storage: the list owning row i
    const float* c = cent + (size_t)l * d;
    float t = 0.f;
    for (int m = 0; m < M; m++) {
        const float* p = codebooks + ((size_t)m * ksub + dfx_pq_code<NB>(codes, i, M, m)) * dsub;
        float ipcp = 0.f, ippp = 0.f;
        for (int tt = 0; tt < dsub; tt++) ipcp = __fmaf_rn(c[m * dsub + tt], p[tt], ipcp);
        for (int tt = 0; tt < dsub; tt++) ippp = __fmaf_rn(p[tt], p[tt], ippp);
        float tm = __fmaf_rn(2.f, ipcp, ippp);
        t = t + tm;
    }
    tvals[i] = t;
}

__global__ void sq_encode_kernel(const float* __restrict__ x, const float* __restrict__ cent,
                                 const int32_t* __restrict__ assign, int64_t n, int d,
                                 __half* __restrict__ codes) {
    int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= n * d) return;
    int64_t i = t / d;
    int c = (int)(t - i * d);
    codes[t] = __float2half_rn(x[t] - cent[(size_t)assign[i] * d + c]);
}

// IVF-SQ8 encode (faiss QT_8bit, non-uniform, by_residual; DESIGN.md section 2): per component
// t = (r - vmin) / vdiff clamped to [0, 1] (0 where vdiff == 0), code = (int)(255 t), truncated
__global__ void sq8_encode_kernel(const float* __restrict__ x, const float* __restrict__ cent,
                                  const int32_t* __restrict__ assign, int64_t n, int d,
                                  const float* __restrict__ trained, uint8_t* __restrict__ codes) {
    int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= n * d) return;
    int64_t i = t / d;
    int c = (int)(t - i * d);
    const float r = x[t] - cent[(size_t)assign[i] * d + c];
    const float vmin = trained[c], vdiff = trained[d + c];
    float u = 0.f;
    if (vdiff != 0.f) {
        u = dfx_div_rn(r - vmin, vdiff);
        u = u < 0.f ? 0.f : u;
        u = u > 1.f ? 1.f : u;
    }
    codes[t] = (uint8_t)(int)(255.f * u);
}

// IVF-SQ8 training: per-dimension min / max of n residual rows.  Pass 1: extrema of chunks of
// `rows_per` rows (grid.y = chunk); pass 2: over the chunks, trained = [vmin, vmax - vmin].
// min and max do not depend on the order, so the result is exact.
__global__ void sq8_minmax_partial_kernel(const float* __restrict__ r, int64_t n, int d, int64_t rows_per,
                                          float* __restrict__ pmin, float* __restrict__ pmax) {
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= d) return;
    const int64_t r0 = (int64_t)blockIdx.y * rows_per;
    const int64_t r1 = min(n, r0 + rows_per);
    float lo = FLT_MAX, hi = -FLT_MAX;
    for (int64_t i = r0; i < r1; i++) {
        const float v = r[i * d + c];
        lo = v < lo ? v : lo;
        hi = v > hi ? v : hi;
    }
    pmin[(int64_t)blockIdx.y * d + c] = lo;
    pmax[(int64_t)blockIdx.y * d + c] = hi;
}
__global__ void sq8_minmax_final_kernel(const float* __restrict__ pmin, const float* __restrict__ pmax,
                                        int64_t nchunks, int d, float* __restrict__ trained) {
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= d) return;
    float lo = FLT_MAX, hi = -FLT_MAX;
    for (int64_t j = 0; j < nchunks; j++) {
        const float a = pmin[j * d + c], b = pmax[j * d + c];
        lo = a < lo ? a : lo;
        hi = b > hi ? b : hi;
    }
    trained[c] = lo;
    trained[d + c] = hi - lo;
}

// list id of every row of the list-sorted storage
__global__ void expand_lists_kernel(const int64_t* __restrict__ list_off, int64_t nlist, int64_t n,
                                    int32_t* __restrict__ out) {
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    out[i] = (int32_t)dfx_list_of(list_off, nlist, i);
}

// new[i] = (src < n_sorted ? old_sorted[src] : pending[src - n_sorted]) in 4-byte words
__global__ void gather_words_kernel(const uint32_t* __restrict__ a, const uint32_t* __restrict__ b,
                                    int64_t n_a, const int32_t* __restrict__ order, int64_t n,
                                    int words, uint32_t* __restrict__ out) {
    int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= n * words) return;
    int64_t i = t / words;
    int w = (int)(t - i * words);
    int64_t src = order[i];
    out[t] = (src < n_a) ? a[src * words + w] : b[(src - n_a) * words + w];
}
__global__ void gather_ids_kernel(const int32_t* __restrict__ old_ids, int64_t n_a,
                                  const int32_t* __restrict__ order, int64_t n,
                                  int32_t* __restrict__ out) {
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    int64_t src = order[i];
    out[i] = (src < n_a) ? old_ids[src] : (int32_t)src;  // pending row j gets id n_a + j == src
}
__global__ void widen_kernel(const int32_t* __restrict__ in, int64_t n, int64_t* __restrict__ out) {
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) out[i] = in[i];
}

static inline unsigned blocks_for(int64_t n, int t) { return (unsigned)dfx_ceil_div(n, t); }

// codes u8[n][M], one per byte: the nearest codeword of each sub-vector of the residual x - c
// (res; c = cent[assign[i]]) or of the row x itself (!res: cent and assign are not read).  The
// kernel keeps the sub-vector in registers for the common dsub (6: d = 768 with M = 128, residual
// codes only); any other dsub runs the generic DS = 0.
static void launch_pq_encode(bool res, const float* x, const float* cent, const int32_t* assign, int64_t n, int d,
                             int M, int ksub, int dsub, const float* codebooks, uint8_t* codes, cudaStream_t st) {
    if (n <= 0) return;
    const dim3 grid(blocks_for(n, 256), (unsigned)M);
    auto launch = [&](auto DS, auto RES) {
        auto kern = pq_encode_kernel<decltype(DS)::value, decltype(RES)::value>;
        DFX_LAUNCH(kern, grid, 256, (size_t)ksub * dsub * 4, st, x, cent, assign, n, d, M, ksub, dsub, codebooks,
                   codes);
    };
    if (res) {
        if (!dispatch_int(IntList<2, 4, 6, 8, 16>{}, dsub, [&](auto DS) { launch(DS, std::true_type{}); }))
            launch(std::integral_constant<int, 0>{}, std::true_type{});
    } else if (!dispatch_int(IntList<2, 4, 8, 16>{}, dsub, [&](auto DS) { launch(DS, std::false_type{}); })) {
        launch(std::integral_constant<int, 0>{}, std::false_type{});
    }
}

// k distinct rows of x f32[n][d] chosen at random (a partial Fisher-Yates shuffle of 0..n-1 driven by
// mt19937_64(seed)) -> out f32[k][d]
static void gather_random_rows(const float* x, int64_t n, int d, int64_t k, uint64_t seed, float* out,
                               cudaStream_t st) {
    std::vector<int32_t> perm((size_t)n);
    std::iota(perm.begin(), perm.end(), 0);
    std::mt19937_64 rng(seed);
    for (int64_t i = 0; i < k; i++) {
        int64_t j = i + (int64_t)(rng() % (uint64_t)(n - i));
        std::swap(perm[(size_t)i], perm[(size_t)j]);
    }
    DevBuf d_sel;
    d_sel.reserve((size_t)k * 4);
    DFX_CUDA(cudaMemcpyAsync(d_sel.p, perm.data(), (size_t)k * 4, cudaMemcpyHostToDevice, st));
    DFX_LAUNCH(gather_rows_kernel, blocks_for(k * d, 256), 256, 0, st, x, d_sel.as<int32_t>(), k, d, 0, d, out);
    DFX_CUDA(cudaStreamSynchronize(st));  // perm is on the stack of this call
}

// Rows grouped by an int32 key in [0, nkeys): run(keys) leaves cnt[key] = rows per key, off = the
// exclusive prefix sum of cnt (nkeys + 1 entries) and order = the row indices sorted by key (a
// stable radix sort, so rows keep ascending order inside a key).  The buffers and cub's temporary
// storage are sized once for n rows; run() may be repeated on new keys.
struct KeyBuckets {
    int64_t n, nkeys;
    int bits = 1;
    DevBuf keys_out, order_in, order, cnt, off, tmp;
    KeyBuckets(int64_t n_, int64_t nkeys_, cudaStream_t st) : n(n_), nkeys(nkeys_) {
        keys_out.reserve((size_t)n * 4);
        order_in.reserve((size_t)n * 4);
        order.reserve((size_t)n * 4);
        cnt.reserve((size_t)(nkeys + 1) * 4);
        off.reserve((size_t)(nkeys + 1) * 4);
        DFX_LAUNCH(iota_kernel, blocks_for(n, 256), 256, 0, st, order_in.as<int32_t>(), n);
        while ((1ll << bits) < nkeys) bits++;
        size_t tmp_sort = 0, tmp_scan = 0;
        cub::DeviceRadixSort::SortPairs(nullptr, tmp_sort, (const int32_t*)nullptr, keys_out.as<int32_t>(),
                                        order_in.as<int32_t>(), order.as<int32_t>(), (int)n, 0, bits, st);
        cub::DeviceScan::ExclusiveSum(nullptr, tmp_scan, cnt.as<int32_t>(), off.as<int32_t>(), (int)(nkeys + 1), st);
        tmp.reserve(std::max(tmp_sort, tmp_scan));
    }
    void run(const int32_t* keys, cudaStream_t st) {
        DFX_CUDA(cudaMemsetAsync(cnt.p, 0, (size_t)(nkeys + 1) * 4, st));
        DFX_LAUNCH(count_kernel, blocks_for(n, 256), 256, 0, st, keys, n, cnt.as<int32_t>());
        size_t tb = tmp.cap;
        DFX_CUDA(cub::DeviceScan::ExclusiveSum(tmp.p, tb, cnt.as<int32_t>(), off.as<int32_t>(), (int)(nkeys + 1),
                                               st));
        tb = tmp.cap;
        DFX_CUDA(cub::DeviceRadixSort::SortPairs(tmp.p, tb, keys, keys_out.as<int32_t>(), order_in.as<int32_t>(),
                                                 order.as<int32_t>(), (int)n, 0, bits, st));
        g_dfx_launches.fetch_add(2, std::memory_order_relaxed);
    }
};

// ------------------------------------------------------------------ assign
void dfx_assign_impl(dfx_index* idx, const float* d_cent, const float* d_cnorm, int64_t nlist,
                     int metric, int d, int64_t n, const float* d_x, int32_t* d_assign,
                     cudaStream_t st) {
    if (n <= 0) return;
    if (idx->tc_enabled && dfx_tc_supported(d) && nlist >= 1024) {
        dfx_tc_assign(idx, d, d_cent, d_cnorm, nlist, metric, n, d_x, d_assign, st);
        return;
    }
    idx->w_best.reserve((size_t)n * 8);
    dfx_launch_assign_fused(d_x, n, d_cent, d_cnorm, nlist, d, metric,
                            idx->w_best.as<unsigned long long>(), d_assign, st);
}

// ------------------------------------------------------------------ k-means on device
static void kmeans_device(dfx_index* idx, int d, int64_t n, const float* d_x, int64_t k, int niter,
                          uint64_t seed, float* d_cent, cudaStream_t st) {
    DFX_REQUIRE(n >= k, "k-means: need at least as many training points as centroids (" +
                            std::to_string(n) + " < " + std::to_string(k) + ")");
    DFX_REQUIRE(n < (1ll << 31), "k-means: too many training points");
    gather_random_rows(d_x, n, d, k, seed, d_cent, st);  // init = random subset without replacement

    DevBuf d_assign, d_cnorm;
    d_assign.reserve((size_t)n * 4);
    d_cnorm.reserve((size_t)k * 4);
    KeyBuckets b(n, k, st);
    std::vector<int32_t> h_cnt((size_t)k + 1);

    for (int it = 0; it < niter; it++) {
        dfx_launch_row_norms(d_cent, k, d, d_cnorm.as<float>(), st);
        dfx_assign_impl(idx, d_cent, d_cnorm.as<float>(), k, DFX_METRIC_L2, d, n, d_x,
                        d_assign.as<int32_t>(), st);
        b.run(d_assign.as<int32_t>(), st);
        int threads = d >= 128 ? 128 : (d >= 64 ? 64 : 32);
        DFX_LAUNCH(centroid_update_kernel, (unsigned)k, threads, 0, st, d_x, d, b.order.as<int32_t>(),
                   b.off.as<int32_t>(), d_cent);
        // empty clusters: split the currently largest (host decides, like the oracle)
        DFX_CUDA(cudaMemcpyAsync(h_cnt.data(), b.cnt.p, (size_t)k * 4, cudaMemcpyDeviceToHost, st));
        DFX_CUDA(cudaStreamSynchronize(st));
        for (int64_t c = 0; c < k; c++) {
            if (h_cnt[(size_t)c] != 0) continue;
            int64_t big = std::max_element(h_cnt.begin(), h_cnt.begin() + k) - h_cnt.begin();
            if (h_cnt[(size_t)big] < 2) break;
            DFX_LAUNCH(split_cluster_kernel, blocks_for(d, 128), 128, 0, st, d_cent, d, (int)c, (int)big);
            h_cnt[(size_t)c] = h_cnt[(size_t)big] / 2;
            h_cnt[(size_t)big] -= h_cnt[(size_t)c];
        }
    }
    DFX_CUDA(cudaStreamSynchronize(st));
}

// ------------------------------------------------------------------ train
// the coarse quantizer from the k-means sample xt f32[nt][d]: centroids, their norms and the
// tensor-core screening table
static void train_coarse(dfx_index* idx, int64_t nt, const float* xt, int niter, cudaStream_t st) {
    const int d = idx->cfg.d;
    const int64_t nlist = idx->cfg.nlist;
    idx->centroids.reserve((size_t)nlist * d * 4);
    idx->cnorm.reserve((size_t)nlist * 4);
    kmeans_device(idx, d, nt, xt, nlist, niter, idx->train_seed, idx->centroids.as<float>(), st);
    dfx_launch_row_norms(idx->centroids.as<float>(), nlist, d, idx->cnorm.as<float>(), st);
    dfx_tc_prepare_centroids(idx, st);
}

// residuals r = x - c of the rows x f32[ns][d], c the nearest coarse centroid under the index's
// metric -> res f32[ns][d]
static void sample_residuals(dfx_index* idx, const float* x, int64_t ns, DevBuf& res, cudaStream_t st) {
    const int d = idx->cfg.d;
    DevBuf assign;
    assign.reserve((size_t)ns * 4);
    res.reserve((size_t)ns * d * 4);
    dfx_assign_impl(idx, idx->centroids.as<float>(), idx->cnorm.as<float>(), idx->cfg.nlist, idx->cfg.metric, d, ns,
                    x, assign.as<int32_t>(), st);
    DFX_LAUNCH(residual_kernel, blocks_for(ns * d, 256), 256, 0, st, x, idx->centroids.as<float>(),
               assign.as<int32_t>(), ns, d, res.as<float>());
}

// the M sub-quantizers of a PQ: sub-quantizer m is k-means (ksub centroids, seed seed0 + m) on
// column slice m of rows f32[ns][ld], into out[m] f32[ksub][dsub]
static void train_subquantizers(dfx_index* idx, const float* rows, int64_t ns, int ld, int M, int ksub, int dsub,
                                int niter, uint64_t seed0, float* out, cudaStream_t st) {
    DevBuf subv;
    subv.reserve((size_t)ns * dsub * 4);
    for (int m = 0; m < M; m++) {
        DFX_LAUNCH(gather_rows_kernel, blocks_for(ns * dsub, 256), 256, 0, st, rows, (const int32_t*)nullptr, ns, dsub,
                   m * dsub, ld, subv.as<float>());
        kmeans_device(idx, dsub, ns, subv.as<float>(), ksub, niter, seed0 + m, out + (size_t)m * ksub * dsub, st);
    }
}

// the codec of the kind, trained on the first rows of the k-means sample xt f32[nt][d] (FLAT_PQ: of the
// training rows themselves)
static void train_codec(dfx_index* idx, int64_t nt, const float* xt, int niter, cudaStream_t st) {
    const int kind = idx->cfg.kind, d = idx->cfg.d;
    const uint64_t seed = idx->train_seed;
    if (idx->has_pq()) {
        // faiss ProductQuantizer on the first min(nt, 256 * ksub) rows: their residuals (IVF_PQ,
        // IVF_PQR), or the raw sub-vectors (FastScan is not by_residual; FLAT_PQ has no lists)
        const int M = idx->M, ksub = idx->ksub, dsub = idx->dsub;
        const int64_t ns = std::min<int64_t>(nt, 256ll * ksub);
        DFX_REQUIRE(ns >= ksub, "train: need at least " + std::to_string(ksub) + " vectors for PQ");
        DevBuf res;
        if (idx->pq_res()) sample_residuals(idx, xt, ns, res, st);
        const float* rows = idx->pq_res() ? res.as<float>() : xt;
        idx->codebooks.reserve((size_t)M * ksub * dsub * 4);
        idx->cbT_valid = false;
        train_subquantizers(idx, rows, ns, d, M, ksub, dsub, niter, seed + 1, idx->codebooks.as<float>(), st);
        if (kind == DFX_IVF_PQR) {
            // faiss IndexIVFPQR::train_encoder: the refinement PQ is trained on what PQ1 leaves of the
            // same residuals, r2 = r - decode(encode(r)); seeds seed + 1 + M + m2 (PQ1 has seed + 1 + m)
            const int M2 = idx->M2, dsub2 = idx->dsub2;
            DevBuf codes, r2;
            codes.reserve((size_t)ns * M);
            r2.reserve((size_t)ns * d * 4);
            launch_pq_encode(false, rows, nullptr, nullptr, ns, d, M, ksub, dsub, idx->codebooks.as<float>(),
                             codes.as<uint8_t>(), st);
            DFX_LAUNCH(pq_residual2_kernel, blocks_for(ns * d, 256), 256, 0, st, rows, (const float*)nullptr,
                       (const int32_t*)nullptr, codes.as<uint8_t>(), ns, d, M, dsub, idx->codebooks.as<float>(),
                       r2.as<float>());
            idx->refine_cb.reserve((size_t)M2 * 256 * dsub2 * 4);
            train_subquantizers(idx, r2.as<float>(), ns, d, M2, 256, dsub2, niter, seed + 1 + M,
                                idx->refine_cb.as<float>(), st);
        }
    } else if (kind == DFX_IVF_SQ8) {
        // faiss ScalarQuantizer (QT_8bit, RS_minmax) on the residuals of the first min(nt, 100000)
        // rows of the k-means sample, the way the PQ above takes a prefix of it
        const int64_t ns = std::min<int64_t>(nt, 100000);
        const int64_t rows_per = 256;
        const int64_t nch = dfx_ceil_div(ns, rows_per);
        DevBuf res, part;
        sample_residuals(idx, xt, ns, res, st);
        part.reserve((size_t)nch * d * 8);
        float* pmin = part.as<float>();
        float* pmax = pmin + (size_t)nch * d;
        DFX_LAUNCH(sq8_minmax_partial_kernel, dim3(blocks_for(d, 128), (unsigned)nch), 128, 0, st,
                   res.as<float>(), ns, d, rows_per, pmin, pmax);
        idx->sq_trained.reserve((size_t)2 * d * 4);
        DFX_LAUNCH(sq8_minmax_final_kernel, blocks_for(d, 128), 128, 0, st, pmin, pmax, nch, d,
                   idx->sq_trained.as<float>());
        DFX_CUDA(cudaStreamSynchronize(st));
    }
}

// an empty, trained index
static void start_empty_lists(dfx_index* idx, cudaStream_t st) {
    const int64_t nlist = idx->cfg.nlist;
    idx->h_list_off.assign((size_t)nlist + 1, 0);
    idx->update_list_lengths();
    idx->list_off.reserve((size_t)(nlist + 1) * 8);
    DFX_CUDA(cudaMemsetAsync(idx->list_off.p, 0, (size_t)(nlist + 1) * 8, st));
    DFX_CUDA(cudaStreamSynchronize(st));
    idx->n_sorted = 0;
    idx->n_pending = 0;
    idx->trained = true;
    dfx_layout_changed(idx, st);
}

void dfx_train_impl(dfx_index* idx, int64_t n, const float* d_x, cudaStream_t st) {
    if (idx->flat_rows()) {  // trained at creation, as faiss's IndexFlat and IndexScalarQuantizer(QT_fp16)
        idx->trained = true;
        return;
    }
    const int d = idx->cfg.d;
    const int64_t nlist = idx->cfg.nlist;
    const int niter = idx->kmeans_niter > 0 ? idx->kmeans_niter : 25;
    if (!idx->is_ivf()) {  // FLAT_PQ (faiss IndexPQ::train): the codebooks alone, and an empty index
        train_codec(idx, n, d_x, niter, st);
        idx->n_sorted = 0;
        idx->trained = true;
        return;
    }
    DFX_REQUIRE(n >= nlist, "train: need at least nlist=" + std::to_string(nlist) +
                                " training vectors, got " + std::to_string(n));

    // faiss Clustering: at most 256 points per centroid (random subset)
    const int64_t nt = std::min<int64_t>(n, (int64_t)idx->max_points_per_centroid * nlist);
    const float* xt = d_x;
    DevBuf sub;
    if (nt < n) {
        sub.reserve((size_t)nt * d * 4);
        gather_random_rows(d_x, n, d, nt, idx->train_seed ^ 0x5bd1e995u, sub.as<float>(), st);
        xt = sub.as<float>();
    }
    train_coarse(idx, nt, xt, niter, st);
    train_codec(idx, nt, xt, niter, st);
    start_empty_lists(idx, st);
}

// ------------------------------------------------------------------ add
static void ensure_pending(dfx_index* idx, int64_t need, cudaStream_t st) {
    if (need <= idx->p_cap) return;
    int64_t cap = std::max<int64_t>(need, idx->p_cap * 2);
    if (idx->reserve_hint > idx->n_sorted)
        cap = std::max<int64_t>(cap, std::min<int64_t>(idx->reserve_hint - idx->n_sorted, need * 64));
    const size_t rb = idx->row_bytes();
    idx->p_list.reserve((size_t)cap * 4, (size_t)idx->n_pending * 4, st);
    idx->p_payload.reserve((size_t)cap * rb, (size_t)idx->n_pending * rb, st);
    if (idx->pq_res())
        idx->p_tvals.reserve((size_t)cap * 4, (size_t)idx->n_pending * 4, st);
    idx->p_cap = cap;
}

// FLAT_SQ16 encode (faiss QT_fp16 without a residual): code = fp16(x), round to nearest even,
// overflow to +-inf
__global__ void f16_encode_kernel(const float* __restrict__ x, int64_t n, __half* __restrict__ codes) {
    const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t < n) codes[t] = __float2half_rn(x[t]);
}

// FLAT / FLAT_SQ16 / FLAT_PQ: the rows (fp32, their fp16 codes, or their PQ codes) in arrival order, and
// under FLAT / FLAT_SQ16 L2 the norms of the stored rows
static void add_flat(dfx_index* idx, int64_t n, const float* d_x, cudaStream_t st) {
    const int d = idx->cfg.d;
    const int64_t N = idx->n_sorted;
    const size_t rb = idx->row_bytes();
    const bool norms = idx->flat_rows() && idx->cfg.metric == DFX_METRIC_L2;
    DFX_REQUIRE(idx->trained || idx->flat_rows(), "add: index is not trained");
    if ((size_t)(N + n) * rb > idx->payload.cap) {
        int64_t cap = std::max<int64_t>({N + n, 2 * N, idx->reserve_hint});
        idx->payload.reserve((size_t)cap * rb, (size_t)N * rb, st);
        if (norms) idx->xnorm.reserve((size_t)cap * 4, (size_t)N * 4, st);
    }
    if (idx->cfg.kind == DFX_FLAT_PQ)
        launch_pq_encode(false, d_x, nullptr, nullptr, n, d, idx->M, idx->ksub, idx->dsub, idx->codebooks.as<float>(),
                         idx->payload.as<uint8_t>() + N * idx->M, st);
    else if (idx->cfg.kind == DFX_FLAT_SQ16)
        DFX_LAUNCH(f16_encode_kernel, blocks_for(n * d, 256), 256, 0, st, d_x, n * d, idx->payload.as<__half>() + N * d);
    else
        DFX_CUDA(cudaMemcpyAsync(idx->payload.as<float>() + N * d, d_x, (size_t)n * d * 4,
                                 cudaMemcpyDeviceToDevice, st));
    if (norms)
        dfx_with_flat_rows(idx, [&](auto rows) { dfx_launch_row_norms(rows + N * d, n, d, idx->xnorm.as<float>() + N, st); });
    idx->n_sorted += n;
}

// the pending list rows (prow, row_bytes() each) of n new vectors x whose lists are plist
static void encode_rows(dfx_index* idx, int64_t n, const float* d_x, const int32_t* plist, unsigned char* prow,
                        cudaStream_t st) {
    const int kind = idx->cfg.kind, d = idx->cfg.d;
    if (kind == DFX_IVF_FLAT) {
        DFX_CUDA(cudaMemcpyAsync(prow, d_x, (size_t)n * d * 4, cudaMemcpyDeviceToDevice, st));
    } else if (idx->has_pq()) {
        // one code per byte first; 4-bit codes are packed afterwards (two sub-quantizers share a
        // byte, so the per-sub-quantizer encode launch cannot write nibbles in place).  FastScan codes
        // the raw vector and keeps no t-value.
        const int M = idx->M, ksub = idx->ksub, dsub = idx->dsub;
        DevBuf unpacked;
        uint8_t* enc = (uint8_t*)prow;
        if (ksub == 16) {
            unpacked.reserve((size_t)n * M);
            enc = unpacked.as<uint8_t>();
        }
        launch_pq_encode(idx->pq_res(), d_x, idx->centroids.as<float>(), plist, n, d, M, ksub, dsub,
                         idx->codebooks.as<float>(), enc, st);
        if (idx->pq_res())
            DFX_LAUNCH(pq_tvals_kernel<8>, blocks_for(n, 128), 128, 0, st, (const uint8_t*)enc, plist,
                       (const int64_t*)nullptr, idx->cfg.nlist, n, d, M, ksub, dsub, idx->codebooks.as<float>(),
                       idx->centroids.as<float>(), idx->p_tvals.as<float>() + idx->n_pending);
        if (ksub == 16)
            DFX_LAUNCH(pq_pack4_kernel, blocks_for(n * M / 2, 256), 256, 0, st, (const uint8_t*)enc,
                       n * M / 2, (uint8_t*)prow);
        // (`unpacked` is freed on return: cudaFree waits for the kernels above)
    } else if (kind == DFX_IVF_SQ16) {
        DFX_LAUNCH(sq_encode_kernel, blocks_for(n * d, 256), 256, 0, st, d_x, idx->centroids.as<float>(),
                   plist, n, d, (__half*)prow);
    } else {  // IVF_SQ8
        DFX_LAUNCH(sq8_encode_kernel, blocks_for(n * d, 256), 256, 0, st, d_x, idx->centroids.as<float>(),
                   plist, n, d, idx->sq_trained.as<float>(), (uint8_t*)prow);
    }
}

// rows id0 .. id0 + n - 1 of a store kept in id order next to the lists (refine_codes of IVF_PQR,
// refine_vecs of the flat refinement), grown to refine_cap rows; returns the first of them
static unsigned char* append_by_id(dfx_index* idx, DevBuf& store, size_t row_bytes, int64_t id0, int64_t n,
                                   cudaStream_t st) {
    if (id0 + n > idx->refine_cap) {
        const int64_t cap = std::max<int64_t>({id0 + n, 2 * idx->refine_cap, idx->reserve_hint});
        store.reserve((size_t)cap * row_bytes, (size_t)id0 * row_bytes, st);
        idx->refine_cap = cap;
    }
    return store.as<unsigned char>() + (size_t)id0 * row_bytes;
}

// the stores by id: the new rows get the ids ntotal .. ntotal + n - 1, their arrival order, so they
// append.  IVF_PQR: refine_codes[id] = refine_pq.encode((x - c) - PQ1(code)), codes1 the PQ1 codes
// just encoded; flat refinement: the raw rows.
static void add_by_id(dfx_index* idx, int64_t n, const float* d_x, const int32_t* plist, const uint8_t* codes1,
                      cudaStream_t st) {
    const int d = idx->cfg.d;
    const int64_t id0 = idx->ntotal();
    if (idx->cfg.kind == DFX_IVF_PQR) {
        uint8_t* rcodes = append_by_id(idx, idx->refine_codes, (size_t)idx->M2, id0, n, st);
        DevBuf r2;
        r2.reserve((size_t)n * d * 4);
        DFX_LAUNCH(pq_residual2_kernel, blocks_for(n * d, 256), 256, 0, st, d_x, idx->centroids.as<float>(), plist,
                   codes1, n, d, idx->M, idx->dsub, idx->codebooks.as<float>(), r2.as<float>());
        launch_pq_encode(false, r2.as<float>(), nullptr, nullptr, n, d, idx->M2, 256, idx->dsub2,
                         idx->refine_cb.as<float>(), rcodes, st);
        // (`r2` is freed on return: cudaFree waits for the kernels above)
    }
    if (idx->rflat()) {
        const size_t rowb = (size_t)d * 4;
        DFX_CUDA(cudaMemcpyAsync(append_by_id(idx, idx->refine_vecs, rowb, id0, n, st), d_x, (size_t)n * rowb,
                                 cudaMemcpyDeviceToDevice, st));
    }
}

void dfx_add_impl(dfx_index* idx, int64_t n, const float* d_x, cudaStream_t st) {
    if (n <= 0) return;
    DFX_REQUIRE(idx->ntotal() + n < (1ll << 31), "a shard holds at most 2^31-1 vectors");
    if (idx->is_flat()) {
        add_flat(idx, n, d_x, st);
        return;
    }
    DFX_REQUIRE(idx->trained, "add: index is not trained");
    ensure_pending(idx, idx->n_pending + n, st);
    int32_t* plist = idx->p_list.as<int32_t>() + idx->n_pending;
    dfx_assign_impl(idx, idx->centroids.as<float>(), idx->cnorm.as<float>(), idx->cfg.nlist, idx->cfg.metric,
                    idx->cfg.d, n, d_x, plist, st);
    unsigned char* prow = idx->p_payload.as<unsigned char>() + (size_t)idx->n_pending * idx->row_bytes();
    encode_rows(idx, n, d_x, plist, prow, st);
    add_by_id(idx, n, d_x, plist, prow, st);
    idx->n_pending += n;
}

void dfx_compute_tvals_sorted(dfx_index* idx, cudaStream_t st) {
    const int64_t n = idx->n_sorted;
    idx->tvals.reserve((size_t)std::max<int64_t>(n, 1) * 4);
    if (n == 0) return;
    auto kern = (idx->ksub == 16) ? pq_tvals_kernel<4> : pq_tvals_kernel<8>;
    DFX_LAUNCH(kern, blocks_for(n, 128), 128, 0, st, idx->payload.as<uint8_t>(),
               (const int32_t*)nullptr, idx->list_off.as<int64_t>(), idx->cfg.nlist, n, idx->cfg.d,
               idx->M, idx->ksub, idx->dsub, idx->codebooks.as<float>(), idx->centroids.as<float>(),
               idx->tvals.as<float>());
}

// ------------------------------------------------------------------ finalize: stage -> lists
void dfx_finalize_impl(dfx_index* idx, cudaStream_t st) {
    if (!idx->is_ivf() || idx->n_pending == 0) return;
    if (idx->il) dfx_pq_il_to_rm(idx, st);  // merge happens on the row-major form
    const int64_t na = idx->n_sorted, nb = idx->n_pending, n = na + nb;
    const int64_t nlist = idx->cfg.nlist;
    const size_t rb = idx->row_bytes();
    DFX_REQUIRE(rb % 4 == 0, "row size must be a multiple of 4 bytes");
    DevBuf keys;
    keys.reserve((size_t)n * 4);
    if (na > 0)
        DFX_LAUNCH(expand_lists_kernel, blocks_for(na, 256), 256, 0, st, idx->list_off.as<int64_t>(),
                   nlist, na, keys.as<int32_t>());
    DFX_CUDA(cudaMemcpyAsync(keys.as<int32_t>() + na, idx->p_list.p, (size_t)nb * 4,
                             cudaMemcpyDeviceToDevice, st));
    KeyBuckets b(n, nlist, st);
    b.run(keys.as<int32_t>(), st);
    keys.release();
    b.keys_out.release();
    b.order_in.release();

    // gather into fresh list-sorted storage
    DevBuf new_payload, new_ids, new_tvals;
    new_payload.reserve((size_t)n * rb);
    new_ids.reserve((size_t)n * 4);
    const int words = (int)(rb / 4);
    DFX_LAUNCH(gather_words_kernel, blocks_for(n * words, 256), 256, 0, st, idx->payload.as<uint32_t>(),
               idx->p_payload.as<uint32_t>(), na, b.order.as<int32_t>(), n, words,
               new_payload.as<uint32_t>());
    DFX_LAUNCH(gather_ids_kernel, blocks_for(n, 256), 256, 0, st, idx->ids.as<int32_t>(), na,
               b.order.as<int32_t>(), n, new_ids.as<int32_t>());
    if (idx->pq_res()) {
        new_tvals.reserve((size_t)n * 4);
        DFX_LAUNCH(gather_words_kernel, blocks_for(n, 256), 256, 0, st, idx->tvals.as<uint32_t>(),
                   idx->p_tvals.as<uint32_t>(), na, b.order.as<int32_t>(), n, 1, new_tvals.as<uint32_t>());
    }
    idx->list_off.reserve((size_t)(nlist + 1) * 8);
    DFX_LAUNCH(widen_kernel, blocks_for(nlist + 1, 256), 256, 0, st, b.off.as<int32_t>(), nlist + 1,
               idx->list_off.as<int64_t>());
    idx->h_list_off.resize((size_t)nlist + 1);
    DFX_CUDA(cudaMemcpyAsync(idx->h_list_off.data(), idx->list_off.p, (size_t)(nlist + 1) * 8,
                             cudaMemcpyDeviceToHost, st));
    DFX_CUDA(cudaStreamSynchronize(st));
    idx->update_list_lengths();
    std::swap(idx->payload, new_payload);
    std::swap(idx->ids, new_ids);
    if (idx->pq_res()) std::swap(idx->tvals, new_tvals);
    idx->p_list.release();
    idx->p_payload.release();
    idx->p_tvals.release();
    idx->p_cap = 0;
    idx->n_sorted = n;
    idx->n_pending = 0;
    // IVF-PQ, M == 32: interleaved blocks for the scan, a layout change of its own
    if (dfx_il_wanted(idx)) dfx_pq_rm_to_il(idx, st);
    else dfx_layout_changed(idx, st);
}

// ------------------------------------------------------------------ reconstruct
__global__ void invert_ids_kernel(const int32_t* __restrict__ ids, int64_t n, int32_t* __restrict__ inv) {
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n && ids[i] >= 0) inv[ids[i]] = (int32_t)i;
}

// Row decoders of reconstruct_kernel: dec(k, id, pos, l) is component k of the vector with local id
// `id`, stored at position pos of list l.  kFrom is what the kernel looks up first: Id, rows
// addressed by id (pos = id); Pos, the storage position pos = inv[id]; List, also the list l that
// holds it (the decoders that add the list's centroid).
enum class RowFrom { Id, Pos, List };

template <RowFrom FROM, class T = float>
struct RowsDec {  // FLAT and the flat refinement (by id), IVF_FLAT (by position): the stored row;
    static constexpr RowFrom kFrom = FROM;  // FLAT_SQ16 (T = __half, by id): the decoded fp16 row
    const T* rows;
    int d;
    __device__ float operator()(int k, int64_t, int64_t pos, int64_t) const { return dfx_elem_f32(rows[pos * d + k]); }
};

struct Sq16Dec {  // IVF_SQ16: c + r in fp16
    static constexpr RowFrom kFrom = RowFrom::List;
    const __half* codes;
    const float* cent;
    int d;
    __device__ float operator()(int k, int64_t, int64_t pos, int64_t l) const {
        return cent[(size_t)l * d + k] + __half2float(codes[pos * d + k]);
    }
};

struct Sq8Dec {  // IVF_SQ8: c + the decode of the list scan (DESIGN.md section 2)
    static constexpr RowFrom kFrom = RowFrom::List;
    const uint8_t* codes;
    const float* cent;
    const float* trained;
    int d;
    __device__ float operator()(int k, int64_t, int64_t pos, int64_t l) const {
        const float t = __fmaf_rn((float)codes[pos * d + k], DFX_SQ8_SCALE, DFX_SQ8_BIAS);
        return cent[(size_t)l * d + k] + __fmaf_rn(t, trained[d + k], trained[k]);
    }
};

// IVF_PQ: c + P[m][code_m].  NB = bits per code of the row-major form (dfx_pq_code); il != 0: the
// codes are the interleaved blocks (dfx_il2_byte of block pos / 32) and pos a padded block position.
template <int NB>
struct PqDec {
    static constexpr RowFrom kFrom = RowFrom::List;
    const uint8_t* codes;
    const float* cent;
    const float* codebooks;
    int d, M, ksub, dsub, il;
    __device__ float operator()(int k, int64_t, int64_t pos, int64_t l) const {
        const int m = k / dsub;
        const int code = il ? codes[(pos >> 5) * 1024 + dfx_il2_byte((int)(pos & 31), m)]
                            : dfx_pq_code<NB>(codes, pos, M, m);
        return cent[(size_t)l * d + k] + codebooks[((size_t)m * ksub + code) * dsub + (k - m * dsub)];
    }
};

struct PqFsDec {  // IVF_PQ_FS: P[m][code_m], no centroid (the codes are of the raw vector)
    static constexpr RowFrom kFrom = RowFrom::Pos;
    const uint8_t* codes;
    const float* codebooks;
    int M, dsub;
    __device__ float operator()(int k, int64_t, int64_t pos, int64_t) const {
        const int m = k / dsub;
        return codebooks[((size_t)m * 16 + dfx_pq_code<4>(codes, pos, M, m)) * dsub + (k - m * dsub)];
    }
};

struct PqFlatDec {  // FLAT_PQ: P[m][code_m] of the row stored by id (8-bit codes of the raw vector)
    static constexpr RowFrom kFrom = RowFrom::Id;
    const uint8_t* codes;
    const float* codebooks;
    int M, dsub;
    __device__ float operator()(int k, int64_t, int64_t pos, int64_t) const {
        const int m = k / dsub;
        return codebooks[((size_t)m * 256 + dfx_pq_code<8>(codes, pos, M, m)) * dsub + (k - m * dsub)];
    }
};

// IVF_PQR: (c + P1[m][code_m]) + P2[m2][refine_code_m2], the reconstruction of faiss's IndexIVFPQR;
// the refinement codes are stored by id
struct PqrDec {
    static constexpr RowFrom kFrom = RowFrom::List;
    PqDec<8> pq1;
    const uint8_t* rcodes;
    const float* rcb;
    int M2, dsub2;
    __device__ float operator()(int k, int64_t id, int64_t pos, int64_t l) const {
        const int m2 = k / dsub2;
        return pq1(k, id, pos, l) + rcb[((size_t)m2 * 256 + rcodes[id * M2 + m2]) * dsub2 + (k - m2 * dsub2)];
    }
};

// One CTA per wanted id.  tag < 0: local ids, an unknown one (-1, >= ntotal) gives a NaN row.
// tag >= 0: exchange ids ((shard tag << 40) | local id, see encode_ids_kernel), only the rows this
// shard owns are decoded and every other row of `out` is left untouched.  `off` holds the list
// offsets, or with il != 0 the block offsets (then inv holds padded block positions).
template <class Dec>
__global__ void reconstruct_kernel(Dec dec, int d, int64_t ntotal, int64_t nlist, const int64_t* __restrict__ want,
                                   const int32_t* __restrict__ inv, const int64_t* __restrict__ off, int il,
                                   float* __restrict__ out, int64_t tag) {
    const int64_t r = blockIdx.x;
    int64_t id = want[r];
    if (tag >= 0) {
        if (id < 0 || ((id >> 40) & 0xfffff) != tag) return;
        id &= (1ll << 40) - 1;
    }
    if (id < 0 || id >= ntotal) {
        for (int k = threadIdx.x; k < d; k += blockDim.x) out[r * d + k] = __int_as_float(0x7fc00000);
        return;
    }
    const int64_t pos = Dec::kFrom == RowFrom::Id ? id : inv[id];
    const int64_t l = Dec::kFrom == RowFrom::List ? dfx_list_of(off, nlist, il ? pos >> 5 : pos) : 0;
    for (int k = threadIdx.x; k < d; k += blockDim.x) out[r * d + k] = dec(k, id, pos, l);
}

void dfx_refresh_inv(dfx_index* idx, cudaStream_t st) {
    if (!idx->is_ivf() || idx->inv_valid) return;
    const int64_t nt = idx->n_sorted;
    const int il = idx->il ? 2 : 0;
    idx->inv.reserve((size_t)std::max<int64_t>(nt, 1) * 4);
    const int64_t npos = il ? idx->nblk * 32 : nt;
    if (npos > 0)
        DFX_LAUNCH(invert_ids_kernel, blocks_for(npos, 256), 256, 0, st,
                   il ? idx->il_ids.as<int32_t>() : idx->ids.as<int32_t>(), npos, idx->inv.as<int32_t>());
    idx->inv_valid = true;
}

void dfx_layout_changed(dfx_index* idx, cudaStream_t st) {
    idx->inv_valid = false;
    if (idx->cfg.kind == DFX_IVF_PQR) dfx_refresh_inv(idx, st);
}

void dfx_reconstruct_impl(dfx_index* idx, int64_t n, const int64_t* d_ids, float* d_out,
                          cudaStream_t st, int64_t tag) {
    if (n <= 0) return;
    if (idx->n_pending > 0) dfx_finalize_impl(idx, st);
    const int d = idx->cfg.d, M = idx->M, ksub = idx->ksub, dsub = idx->dsub;
    const int il = idx->il ? 2 : 0;  // 0 = row-major, else the block layout
    const uint8_t* codes = il ? idx->il_codes.as<uint8_t>() : idx->payload.as<uint8_t>();
    const float* cent = idx->centroids.as<float>();
    const float* cb = idx->codebooks.as<float>();
    auto run = [&](auto dec) {
        DFX_LAUNCH(reconstruct_kernel<decltype(dec)>, (unsigned)n, 128, 0, st, dec, d, idx->n_sorted, idx->cfg.nlist,
                   d_ids, idx->inv.as<int32_t>(), il ? idx->blk_off.as<int64_t>() : idx->list_off.as<int64_t>(), il,
                   d_out, tag);
    };
    // flat refinement: the stored row, addressed by id as a FLAT index addresses its rows
    if (idx->rflat()) return run(RowsDec<RowFrom::Id>{idx->refine_vecs.as<float>(), d});
    dfx_refresh_inv(idx, st);
    switch (idx->cfg.kind) {
        case DFX_FLAT: return run(RowsDec<RowFrom::Id>{idx->payload.as<float>(), d});
        case DFX_FLAT_SQ16: return run(RowsDec<RowFrom::Id, __half>{idx->payload.as<__half>(), d});
        case DFX_FLAT_PQ: return run(PqFlatDec{idx->payload.as<uint8_t>(), cb, M, dsub});
        case DFX_IVF_FLAT: return run(RowsDec<RowFrom::Pos>{idx->payload.as<float>(), d});
        case DFX_IVF_SQ16: return run(Sq16Dec{idx->payload.as<__half>(), cent, d});
        case DFX_IVF_SQ8: return run(Sq8Dec{idx->payload.as<uint8_t>(), cent, idx->sq_trained.as<float>(), d});
        case DFX_IVF_PQ:
            if (ksub == 16) return run(PqDec<4>{codes, cent, cb, d, M, ksub, dsub, il});
            return run(PqDec<8>{codes, cent, cb, d, M, ksub, dsub, il});
        case DFX_IVF_PQ_FS: return run(PqFsDec{idx->payload.as<uint8_t>(), cb, M, dsub});
        case DFX_IVF_PQR:
            return run(PqrDec{PqDec<8>{codes, cent, cb, d, M, ksub, dsub, il}, idx->refine_codes.as<uint8_t>(),
                              idx->refine_cb.as<float>(), idx->M2, idx->dsub2});
    }
}
