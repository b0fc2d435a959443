// dfx_api.cu -- extern "C" surface of libdfx.so (include/dfx.h) + synthetic data generator.
#include "dfx_internal.h"
#include <cstdlib>
#include <cstring>
#include <cmath>
#include <vector>

static thread_local std::string g_last_error;
std::atomic<long long> g_dfx_launches{0};

void dfx_set_error(const std::string& msg) { g_last_error = msg; }

#define DFX_API_BEGIN try {
#define DFX_API_END                                   \
    }                                                 \
    catch (const DfxError& e) {                       \
        g_last_error = e.msg;                         \
        return 1;                                     \
    }                                                 \
    catch (const std::exception& e) {                 \
        g_last_error = std::string("dfx: ") + e.what(); \
        return 2;                                     \
    }                                                 \
    return 0;

static void require_device(int device) {
    int n = 0;
    cudaError_t e = cudaGetDeviceCount(&n);
    if (e != cudaSuccess || n <= 0)
        throw DfxError{std::string("libdfx needs a CUDA device (no CPU fallback): ") +
                       (e != cudaSuccess ? cudaGetErrorString(e) : "no device found")};
    DFX_REQUIRE(device >= 0 && device < n, "bad device ordinal " + std::to_string(device));
    cudaDeviceProp p;
    DFX_CUDA(cudaGetDeviceProperties(&p, device));
    DFX_REQUIRE(p.major == 9 && p.minor == 0, std::string("libdfx is built for sm_90a only; device is sm_") +
                                   std::to_string(p.major) + std::to_string(p.minor));
}

// one property of the current device, read once per device ordinal (cache entry 0 = not queried yet)
template <class Get>
static int cached_device_prop(std::atomic<int> (&cache)[64], Get get) {
    int dev = 0;
    DFX_CUDA(cudaGetDevice(&dev));
    DFX_REQUIRE(dev >= 0 && dev < 64, "device ordinal out of range");
    int n = cache[dev].load(std::memory_order_relaxed);
    if (n == 0) {
        cudaDeviceProp p;
        DFX_CUDA(cudaGetDeviceProperties(&p, dev));
        n = get(p);
        cache[dev].store(n, std::memory_order_relaxed);
    }
    return n;
}

int dfx_num_sms() {
    static std::atomic<int> cache[64];
    return cached_device_prop(cache, [](const cudaDeviceProp& p) { return p.multiProcessorCount; });
}

int dfx_smem_optin() {
    static std::atomic<int> cache[64];
    return cached_device_prop(cache, [](const cudaDeviceProp& p) { return (int)p.sharedMemPerBlockOptin; });
}

struct DeviceGuard {
    int prev = -1;
    explicit DeviceGuard(int dev) {
        cudaGetDevice(&prev);
        if (prev != dev) cudaSetDevice(dev);
        else prev = -1;
    }
    ~DeviceGuard() {
        if (prev >= 0) cudaSetDevice(prev);
    }
};

extern "C" {

const char* dfx_last_error(void) { return g_last_error.c_str(); }
#ifndef DFX_SRC_HASH
#define DFX_SRC_HASH "unknown"
#endif
// ends with the hash of the sources the library was compiled from (build.py: source_hash)
const char* dfx_version(void) { return "dfx 0.2 (sm_90a) dfx-src-sha256=" DFX_SRC_HASH; }
int64_t dfx_launch_count(void) { return (int64_t)g_dfx_launches.load(); }
int dfx_debug_il_byte(int layout, int v, int m) { return dfx_il_byte_of(layout, v & 31, m & 31); }
int dfx_debug_tc_screen(dfx_index* idx, int64_t nq, const float* d_x, int npl, float* d_gmin, float* d_gmin2,
                        uint8_t* d_gargc) {
    DFX_API_BEGIN
    DFX_REQUIRE(idx && d_x && d_gmin && d_gmin2 && d_gargc, "null argument");
    DFX_REQUIRE(nq >= 1, "nq must be >= 1");
    DFX_REQUIRE(npl == 1 || npl == 2, "npl must be 1 (FAST) or 2 (PRECISE)");
    DFX_REQUIRE(idx->is_ivf(), "the screening table of an IVF index is its centroids");
    std::lock_guard<std::mutex> lk(idx->mu);
    DeviceGuard g(idx->cfg.device);
    idx->join_dev();
    dfx_tc_debug_screen(idx, nq, d_x, npl, d_gmin, d_gmin2, d_gargc, idx->stream);
    DFX_CUDA(cudaStreamSynchronize(idx->stream));
    DFX_API_END
}

int dfx_create(const dfx_cfg* cfg, dfx_index** out) {
    DFX_API_BEGIN
    DFX_REQUIRE(cfg && out, "null argument");
    DFX_REQUIRE(cfg->kind >= DFX_FLAT && cfg->kind <= DFX_FLAT_PQ, "unknown index kind");
    DFX_REQUIRE(cfg->kind == DFX_IVF_PQR || cfg->refine_m == 0, "refine_m must be 0 for every kind but IVF_PQR");
    DFX_REQUIRE(cfg->metric == DFX_METRIC_IP || cfg->metric == DFX_METRIC_L2,
                "Only dot and l2 metrics are supported.");
    DFX_REQUIRE(cfg->d > 0 && cfg->d <= 4096, "dimension must be in [1, 4096]");
    require_device(cfg->device);
    std::unique_ptr<dfx_index> idx(new dfx_index());
    idx->cfg = *cfg;
    if (cfg->kind == DFX_FLAT_SQ16) {
        // faiss's IndexScalarQuantizer(QT_fp16): no lists, no codebooks, no refinement
        DFX_REQUIRE(cfg->nlist == 0 && cfg->pq_m == 0 && cfg->pq_nbits == 0 && cfg->refine_m == 0 &&
                        cfg->refine_flat == 0,
                    "FLAT_SQ16: nlist, pq_m, pq_nbits, refine_m and refine_flat must be 0 (an fp16 scalar quantizer "
                    "without inverted lists), got nlist=" + std::to_string(cfg->nlist) + ", pq_m=" +
                        std::to_string(cfg->pq_m) + ", pq_nbits=" + std::to_string(cfg->pq_nbits) + ", refine_m=" +
                        std::to_string(cfg->refine_m) + ", refine_flat=" + std::to_string(cfg->refine_flat));
    }
    if (cfg->kind == DFX_FLAT_PQ) {
        // faiss's IndexPQ(d, M, 8, metric): no lists, no refinement; the limits of 8-bit IVF-PQ (one query's
        // fp32 table, M x 256 x 4 B, is staged in one thread block's shared memory)
        DFX_REQUIRE(cfg->nlist == 0 && cfg->refine_m == 0 && cfg->refine_flat == 0,
                    "FLAT_PQ: nlist, refine_m and refine_flat must be 0 (a product quantizer without inverted "
                    "lists), got nlist=" + std::to_string(cfg->nlist) + ", refine_m=" + std::to_string(cfg->refine_m) +
                        ", refine_flat=" + std::to_string(cfg->refine_flat));
        DFX_REQUIRE(cfg->pq_nbits == 8, "FLAT_PQ: 8 bits per sub-quantizer, got " + std::to_string(cfg->pq_nbits));
        DFX_REQUIRE(cfg->pq_m >= 4 && cfg->pq_m <= 128 && cfg->pq_m % 4 == 0 && cfg->d % cfg->pq_m == 0,
                    "FLAT_PQ: the number of sub-quantizers must be a multiple of 4, at most 128, that divides d, "
                    "got M=" + std::to_string(cfg->pq_m) + ", d=" + std::to_string(cfg->d));
        idx->M = cfg->pq_m;
        idx->ksub = 256;
        idx->dsub = cfg->d / cfg->pq_m;
    }
    if (cfg->kind != DFX_FLAT && cfg->kind != DFX_FLAT_SQ16 && cfg->kind != DFX_FLAT_PQ) {
        DFX_REQUIRE(cfg->nlist >= 1 && cfg->nlist < (1ll << 24), "nlist must be in [1, 2^24)");
        DFX_REQUIRE(cfg->d % 4 == 0, "IVF indexes need a dimension that is a multiple of 4");
    }
    if (cfg->kind == DFX_IVF_PQ) {
        DFX_REQUIRE(cfg->pq_nbits == 8 || cfg->pq_nbits == 4,
                    "IVF-PQ: 8 or 4 bits per sub-quantizer are supported, got " + std::to_string(cfg->pq_nbits));
        if (cfg->pq_nbits == 8) {
            DFX_REQUIRE(cfg->pq_m >= 4 && cfg->pq_m % 4 == 0 && cfg->d % cfg->pq_m == 0,
                        "IVF-PQ: the number of sub-quantizers must be a multiple of 4 that divides d");
            DFX_REQUIRE(cfg->pq_m <= 128,
                        "IVF-PQ: at most 128 sub-quantizers are supported (one query's fp32 distance table, "
                        "M x 256 x 4 bytes, must fit in one thread block's shared memory; more would need split "
                        "or fp16 tables, which are not bit-exact)");
        } else {
            // a packed row (M / 2 bytes) is whole 32-bit words, and the scan's register table
            // (M / 2 floats per lane) stays within 64 registers
            DFX_REQUIRE(cfg->pq_m >= 8 && cfg->pq_m <= 128 && cfg->pq_m % 8 == 0 && cfg->d % cfg->pq_m == 0,
                        "IVF-PQ with 4-bit codes: the number of sub-quantizers must be a multiple of 8 in "
                        "[8, 128] that divides d, got M=" + std::to_string(cfg->pq_m) + ", d=" +
                            std::to_string(cfg->d));
        }
        idx->M = cfg->pq_m;
        idx->ksub = 1 << cfg->pq_nbits;
        idx->dsub = cfg->d / cfg->pq_m;
    }
    if (cfg->kind == DFX_IVF_PQ_FS) {
        // the list scan sums 8-bit quantized L2 tables; there is no inner-product table
        DFX_REQUIRE(cfg->metric == DFX_METRIC_L2,
                    "IVF-PQ FastScan: only the L2 metric is supported (for the index and its coarse quantizer)");
        DFX_REQUIRE(cfg->pq_nbits == 4,
                    "IVF-PQ FastScan: 4 bits per sub-quantizer, got " + std::to_string(cfg->pq_nbits));
        DFX_REQUIRE(cfg->pq_m >= 8 && cfg->pq_m <= 128 && cfg->pq_m % 8 == 0 && cfg->d % cfg->pq_m == 0,
                    "IVF-PQ FastScan: the number of sub-quantizers must be a multiple of 8 in [8, 128] that "
                    "divides d, got M=" + std::to_string(cfg->pq_m) + ", d=" + std::to_string(cfg->d));
        idx->M = cfg->pq_m;
        idx->ksub = 16;
        idx->dsub = cfg->d / cfg->pq_m;
    }
    if (cfg->kind == DFX_IVF_PQR) {
        // faiss's factory refuses IVFPQR for inner product; the first stage is the 8-bit IVF-PQ scan
        DFX_REQUIRE(cfg->metric == DFX_METRIC_L2,
                    "IVF-PQR: only the L2 metric is supported (for the index and its coarse quantizer)");
        DFX_REQUIRE(cfg->pq_nbits == 8, "IVF-PQR: 8 bits per sub-quantizer, got " + std::to_string(cfg->pq_nbits));
        DFX_REQUIRE(cfg->pq_m >= 4 && cfg->pq_m <= 128 && cfg->pq_m % 4 == 0 && cfg->d % cfg->pq_m == 0,
                    "IVF-PQR: the number of sub-quantizers must be a multiple of 4, at most 128, that divides d, "
                    "got M=" + std::to_string(cfg->pq_m) + ", d=" + std::to_string(cfg->d));
        DFX_REQUIRE(cfg->refine_m >= 4 && cfg->refine_m <= 128 && cfg->refine_m % 4 == 0 && cfg->d % cfg->refine_m == 0,
                    "IVF-PQR: the number of refinement sub-quantizers must be a multiple of 4, at most 128, that "
                    "divides d, got M2=" + std::to_string(cfg->refine_m) + ", d=" + std::to_string(cfg->d));
        idx->M = cfg->pq_m;
        idx->ksub = 256;
        idx->dsub = cfg->d / cfg->pq_m;
        idx->M2 = cfg->refine_m;
        idx->dsub2 = cfg->d / cfg->refine_m;
    }
    if (cfg->refine_flat) {
        // flat refinement (faiss IndexRefineFlat): exact re-ranking only makes sense over a lossy codec
        DFX_REQUIRE(cfg->kind != DFX_FLAT && cfg->kind != DFX_IVF_FLAT,
                    "refine_flat must be 0 for FLAT and IVF_FLAT: their distances are already exact");
        DFX_REQUIRE(cfg->kind != DFX_IVF_PQR, "refine_flat must be 0 for IVF_PQR: it has its own refinement");
        DFX_REQUIRE(cfg->kind != DFX_IVF_PQ || cfg->pq_nbits == 8,
                    "refine_flat must be 0 for IVF-PQ with 4-bit codes (IVF-PQ FastScan takes it)");
        DFX_REQUIRE(cfg->metric == DFX_METRIC_L2,
                    "flat refinement: only the L2 metric is supported (for the index and its coarse quantizer)");
        idx->k_factor = 1.f;  // faiss IndexRefine default
    }
    DeviceGuard g(cfg->device);
    DFX_CUDA(cudaStreamCreateWithFlags(&idx->stream, cudaStreamNonBlocking));
    *out = idx.release();
    DFX_API_END
}

void dfx_destroy(dfx_index* idx) {
    if (!idx) return;
    {
        DeviceGuard g(idx->cfg.device);
        if (idx->stream) {
            cudaStreamSynchronize(idx->stream);
            cudaStreamDestroy(idx->stream);
        }
        idx->prof_scan.destroy();
        idx->prof_refine.destroy();
        if (idx->tc_stat_ev) cudaEventDestroy(idx->tc_stat_ev);
        if (idx->dev_done) cudaEventDestroy(idx->dev_done);
        if (idx->tc_stat_h) cudaFreeHost(idx->tc_stat_h);
        delete idx;
    }
}

int dfx_set_param(dfx_index* idx, const char* name, double value) {
    DFX_API_BEGIN
    idx->generation++;
    std::string n(name);
    if (n == "kmeans_niter") idx->kmeans_niter = (int)value;
    else if (n == "max_points_per_centroid") idx->max_points_per_centroid = (int)value;
    else if (n == "train_seed") idx->train_seed = (uint64_t)value;
    else if (n == "tensor_cores") idx->tc_enabled = value != 0;
    else if (n == "interleaved") {
        std::lock_guard<std::mutex> lk(idx->mu);
        DeviceGuard g(idx->cfg.device);
        idx->join_dev();
        idx->il_enabled = value != 0;
        if (!idx->il_enabled) dfx_pq_il_to_rm(idx, idx->stream);
        else if (idx->trained && idx->n_pending == 0 && idx->n_sorted > 0) dfx_pq_rm_to_il(idx, idx->stream);
    }
    else if (n == "flat_tensor_cores") idx->flat_tc = value != 0;
    else if (n == "rows_inflight") {
        DFX_REQUIRE(value == 0 || value == 4 || value == 8, "rows_inflight must be 0 (by row size), 4 or 8");
        idx->rows_inflight = (int)value;
    }
    else if (n == "tc_screen_mode") {  // 0 = AUTO, 1 = FAST (one fp16 MMA), 2 = PRECISE (hi/lo split, three MMAs)
        DFX_REQUIRE(value == 0 || value == 1 || value == 2, "tc_screen_mode must be 0 (auto), 1 (fast) or 2 (precise)");
        idx->tc_mode = (int)value;
        idx->tc_fast = value == 1;
        idx->tc_stat_pending = false;
        idx->tc_acc_rows = idx->tc_acc_bad = 0;
    }
    else if (n == "tc_auto_window") {
        DFX_REQUIRE(value >= 1 && value <= (double)(1 << 30), "tc_auto_window must be 1 .. 2^30 rows");
        idx->tc_auto_window = (int64_t)value;
        idx->tc_acc_rows = idx->tc_acc_bad = 0;
    }
    else if (n == "il2_threads") {
        DFX_REQUIRE(value == 0 || value == 256 || value == 512, "il2_threads must be 0 (default), 256 or 512");
        idx->il2_threads = (int)value;
    }
    else if (n == "il2_prefetch") {
        DFX_REQUIRE(value >= -1 && value <= 32, "il2_prefetch must be -1 (default) or 0..32 blocks");
        idx->il2_prefetch = (int)value;
    }
    else if (n == "k_factor") {
        DFX_REQUIRE(idx->cfg.kind == DFX_IVF_PQR || idx->rflat(),
                    "k_factor is a parameter of IVF-PQR indexes and of indexes with a flat refinement");
        DFX_REQUIRE(value >= 1 && value <= 16384, "k_factor must be in [1, 16384]");
        idx->k_factor = (float)value;
    }
    else throw DfxError{"unknown parameter " + n};
    DFX_API_END
}

// the device memory of an index's persistent arrays (dfx_get_param "index_bytes"): everything but the
// search and range-search workspace and the scratch of the screening
static size_t index_bytes(const dfx_index* idx) {
    const DevBuf* held[] = {&idx->centroids, &idx->cnorm, &idx->codebooks, &idx->sq_trained, &idx->list_off,
                            &idx->ids, &idx->payload, &idx->tvals, &idx->xnorm, &idx->p_list, &idx->p_payload,
                            &idx->p_tvals, &idx->inv, &idx->il_codes, &idx->il_tvals, &idx->il_ids, &idx->blk_off,
                            &idx->codebooksT, &idx->tc_tab.planes, &idx->tc_tab.cterm, &idx->tc_tab.mean,
                            &idx->refine_cb, &idx->refine_codes, &idx->refine_vecs};
    size_t b = 0;
    for (const DevBuf* h : held) b += h->cap;
    return b;
}

int dfx_get_param(dfx_index* idx, const char* name, double* value) {
    DFX_API_BEGIN
    DFX_REQUIRE(idx && name && value, "null argument");
    std::string n(name);
    if (n.rfind("tc_stat_", 0) == 0 || n == "tc_fast") {
        DeviceGuard g(idx->cfg.device);
        dfx_tc_stats_sync(idx);  // fold the outstanding launch statistics in (AUTO precision)
    }
    if (n == "kmeans_niter") *value = idx->kmeans_niter;
    else if (n == "max_points_per_centroid") *value = idx->max_points_per_centroid;
    else if (n == "train_seed") *value = (double)idx->train_seed;
    else if (n == "tensor_cores") *value = idx->tc_enabled;
    else if (n == "tc_screen_mode") *value = idx->tc_mode;
    else if (n == "tc_fast") *value = idx->tc_fast;
    else if (n == "tc_auto_window") *value = (double)idx->tc_auto_window;
    else if (n == "tc_cmax2") *value = idx->tc_tab.cmax2;
    else if (n == "tc_cmax2c") *value = idx->tc_tab.cmax2c;
    else if (n == "tc_stat_rows") *value = (double)idx->tc_last_rows;
    else if (n == "tc_stat_overflow") *value = (double)idx->tc_last_overflow;
    else if (n == "tc_stat_fast_would") *value = (double)idx->tc_last_fast_would;
    else if (n == "flat_tensor_cores") *value = idx->flat_tc;
    else if (n == "interleaved") *value = idx->il_enabled;
    else if (n == "il2_threads") *value = idx->il2_threads;
    else if (n == "il2_prefetch") *value = idx->il2_prefetch;
    else if (n == "rows_inflight") *value = idx->rows_inflight;
    else if (n == "workspace_bytes") *value = (double)idx->w_part.cap;  // read-only
    else if (n == "index_bytes") *value = (double)index_bytes(idx);     // read-only
    else if (n == "k_factor" && (idx->cfg.kind == DFX_IVF_PQR || idx->rflat())) *value = idx->k_factor;
    else if (n == "refine_ms" || n == "refine_launches") {  // read-only
        std::lock_guard<std::mutex> lk(idx->mu);
        DeviceGuard g(idx->cfg.device);
        idx->join_dev();
        *value = n == "refine_launches" ? (double)idx->prof_refine.used : idx->prof_refine.sum_ms();
    }
    else throw DfxError{"unknown parameter " + n};
    DFX_API_END
}

int dfx_train_dev(dfx_index* idx, int64_t n, const float* d_x, void* stream) {
    DFX_API_BEGIN
    idx->generation++;
    std::lock_guard<std::mutex> lk(idx->mu);
    DeviceGuard g(idx->cfg.device);
    idx->join_dev_if_other((cudaStream_t)stream);
    dfx_train_impl(idx, n, d_x, (cudaStream_t)stream);
    idx->note_dev((cudaStream_t)stream);
    DFX_API_END
}
int dfx_add_dev(dfx_index* idx, int64_t n, const float* d_x, void* stream) {
    DFX_API_BEGIN
    idx->generation++;
    std::lock_guard<std::mutex> lk(idx->mu);
    DeviceGuard g(idx->cfg.device);
    idx->join_dev_if_other((cudaStream_t)stream);
    dfx_add_impl(idx, n, d_x, (cudaStream_t)stream);
    idx->note_dev((cudaStream_t)stream);
    DFX_API_END
}
int dfx_train(dfx_index* idx, int64_t n, const float* x) {
    DFX_API_BEGIN
    idx->generation++;
    std::lock_guard<std::mutex> lk(idx->mu);
    DeviceGuard g(idx->cfg.device);
    idx->join_dev();
    DevBuf buf;
    buf.reserve((size_t)std::max<int64_t>(n, 1) * idx->cfg.d * 4);
    DFX_CUDA(cudaMemcpyAsync(buf.p, x, (size_t)n * idx->cfg.d * 4, cudaMemcpyHostToDevice, idx->stream));
    dfx_train_impl(idx, n, buf.as<float>(), idx->stream);
    DFX_CUDA(cudaStreamSynchronize(idx->stream));
    DFX_API_END
}
int dfx_add(dfx_index* idx, int64_t n, const float* x) {
    DFX_API_BEGIN
    idx->generation++;
    std::lock_guard<std::mutex> lk(idx->mu);
    DeviceGuard g(idx->cfg.device);
    idx->join_dev();
    const int64_t chunk = 1 << 20;
    DevBuf buf;
    buf.reserve((size_t)std::min<int64_t>(std::max<int64_t>(n, 1), chunk) * idx->cfg.d * 4);
    for (int64_t i0 = 0; i0 < n; i0 += chunk) {
        int64_t c = std::min(chunk, n - i0);
        DFX_CUDA(cudaMemcpyAsync(buf.p, x + i0 * idx->cfg.d, (size_t)c * idx->cfg.d * 4,
                                 cudaMemcpyHostToDevice, idx->stream));
        dfx_add_impl(idx, c, buf.as<float>(), idx->stream);
        DFX_CUDA(cudaStreamSynchronize(idx->stream));
    }
    DFX_API_END
}
int dfx_reserve(dfx_index* idx, int64_t n_total) {
    DFX_API_BEGIN
    idx->reserve_hint = n_total;
    DFX_API_END
}
int dfx_finalize(dfx_index* idx, void* stream) {
    DFX_API_BEGIN
    idx->generation++;
    std::lock_guard<std::mutex> lk(idx->mu);
    DeviceGuard g(idx->cfg.device);
    idx->join_dev();
    cudaStream_t st = stream ? (cudaStream_t)stream : idx->stream;
    dfx_finalize_impl(idx, st);
    DFX_CUDA(cudaStreamSynchronize(st));
    DFX_API_END
}

int dfx_search_dev(dfx_index* idx, int64_t nq, const float* d_x, int64_t k, float* d_D, int64_t* d_I,
                   void* stream) {
    DFX_API_BEGIN
    std::lock_guard<std::mutex> lk(idx->mu);
    DeviceGuard g(idx->cfg.device);
    idx->join_dev_if_other((cudaStream_t)stream);
    dfx_search_impl(idx, nq, d_x, k, d_D, d_I, (cudaStream_t)stream);
    idx->note_dev((cudaStream_t)stream);
    DFX_API_END
}
int dfx_search(dfx_index* idx, int64_t nq, const float* x, int64_t k, float* D, int64_t* I) {
    DFX_API_BEGIN
    std::lock_guard<std::mutex> lk(idx->mu);
    DeviceGuard g(idx->cfg.device);
    idx->join_dev();
    if (nq <= 0) return 0;
    DFX_REQUIRE(k >= 1, "k must be >= 1");
    const int d = idx->cfg.d;
    idx->w_q.reserve((size_t)nq * d * 4);
    idx->w_D.reserve((size_t)nq * k * 4);
    idx->w_I.reserve((size_t)nq * k * 8);
    DFX_CUDA(cudaMemcpyAsync(idx->w_q.p, x, (size_t)nq * d * 4, cudaMemcpyHostToDevice, idx->stream));
    dfx_search_impl(idx, nq, idx->w_q.as<float>(), k, idx->w_D.as<float>(), idx->w_I.as<int64_t>(),
                    idx->stream);
    DFX_CUDA(cudaMemcpyAsync(D, idx->w_D.p, (size_t)nq * k * 4, cudaMemcpyDeviceToHost, idx->stream));
    DFX_CUDA(cudaMemcpyAsync(I, idx->w_I.p, (size_t)nq * k * 8, cudaMemcpyDeviceToHost, idx->stream));
    DFX_CUDA(cudaStreamSynchronize(idx->stream));
    DFX_API_END
}

int dfx_range_search_dev(dfx_index* idx, int64_t nq, const float* d_x, float radius, int64_t* d_lims, int64_t* total,
                         void* stream) {
    DFX_API_BEGIN
    DFX_REQUIRE(idx && d_lims && total, "null argument");
    std::lock_guard<std::mutex> lk(idx->mu);
    DeviceGuard g(idx->cfg.device);
    idx->join_dev_if_other((cudaStream_t)stream);
    dfx_range_impl(idx, nq, d_x, radius, d_lims, total, (cudaStream_t)stream);
    idx->note_dev((cudaStream_t)stream);
    DFX_API_END
}
int dfx_range_fetch_dev(dfx_index* idx, float* d_D, int64_t* d_I, void* stream) {
    DFX_API_BEGIN
    DFX_REQUIRE(idx, "null argument");
    std::lock_guard<std::mutex> lk(idx->mu);
    DeviceGuard g(idx->cfg.device);
    idx->join_dev_if_other((cudaStream_t)stream);
    dfx_range_fetch_impl(idx, d_D, d_I, (cudaStream_t)stream);
    idx->note_dev((cudaStream_t)stream);
    DFX_API_END
}
int dfx_range_search(dfx_index* idx, int64_t nq, const float* x, float radius, int64_t* lims) {
    DFX_API_BEGIN
    DFX_REQUIRE(idx && lims, "null argument");
    DFX_REQUIRE(nq >= 0, "nq must be >= 0");
    std::lock_guard<std::mutex> lk(idx->mu);
    DeviceGuard g(idx->cfg.device);
    idx->join_dev();
    const size_t xb = (size_t)nq * idx->cfg.d * 4;
    idx->w_q.reserve(std::max<size_t>(xb, 4));
    idx->r_lims.reserve((size_t)(nq + 1) * 8);
    if (xb) DFX_CUDA(cudaMemcpyAsync(idx->w_q.p, x, xb, cudaMemcpyHostToDevice, idx->stream));
    int64_t total = 0;
    dfx_range_impl(idx, nq, idx->w_q.as<float>(), radius, idx->r_lims.as<int64_t>(), &total, idx->stream);
    DFX_CUDA(cudaMemcpyAsync(lims, idx->r_lims.p, (size_t)(nq + 1) * 8, cudaMemcpyDeviceToHost, idx->stream));
    DFX_CUDA(cudaStreamSynchronize(idx->stream));
    DFX_API_END
}
int dfx_range_fetch(dfx_index* idx, float* D, int64_t* I) {
    DFX_API_BEGIN
    DFX_REQUIRE(idx, "null argument");
    std::lock_guard<std::mutex> lk(idx->mu);
    DeviceGuard g(idx->cfg.device);
    idx->join_dev();
    const int64_t n = std::max<int64_t>(idx->r_total, 0);
    idx->w_D.reserve((size_t)std::max<int64_t>(n, 1) * 4);
    idx->w_I.reserve((size_t)std::max<int64_t>(n, 1) * 8);
    dfx_range_fetch_impl(idx, idx->w_D.as<float>(), idx->w_I.as<int64_t>(), idx->stream);
    if (n) {
        DFX_CUDA(cudaMemcpyAsync(D, idx->w_D.p, (size_t)n * 4, cudaMemcpyDeviceToHost, idx->stream));
        DFX_CUDA(cudaMemcpyAsync(I, idx->w_I.p, (size_t)n * 8, cudaMemcpyDeviceToHost, idx->stream));
    }
    DFX_CUDA(cudaStreamSynchronize(idx->stream));
    DFX_API_END
}

int dfx_reconstruct(dfx_index* idx, int64_t n, const int64_t* ids, float* out) {
    DFX_API_BEGIN
    std::lock_guard<std::mutex> lk(idx->mu);
    DeviceGuard g(idx->cfg.device);
    idx->join_dev();
    if (n <= 0) return 0;
    DevBuf d_ids, d_out;
    d_ids.reserve((size_t)n * 8);
    d_out.reserve((size_t)n * idx->cfg.d * 4);
    DFX_CUDA(cudaMemcpyAsync(d_ids.p, ids, (size_t)n * 8, cudaMemcpyHostToDevice, idx->stream));
    dfx_reconstruct_impl(idx, n, d_ids.as<int64_t>(), d_out.as<float>(), idx->stream);
    DFX_CUDA(cudaMemcpyAsync(out, d_out.p, (size_t)n * idx->cfg.d * 4, cudaMemcpyDeviceToHost, idx->stream));
    DFX_CUDA(cudaStreamSynchronize(idx->stream));
    DFX_API_END
}

int dfx_reconstruct_dev(dfx_index* idx, int64_t n, const int64_t* d_ids, int64_t shard_tag, float* d_out,
                        void* stream) {
    DFX_API_BEGIN
    std::lock_guard<std::mutex> lk(idx->mu);
    DeviceGuard g(idx->cfg.device);
    idx->join_dev_if_other((cudaStream_t)stream);
    dfx_reconstruct_impl(idx, n, d_ids, d_out, (cudaStream_t)stream, shard_tag);
    idx->note_dev((cudaStream_t)stream);
    DFX_API_END
}

int dfx_set_nprobe(dfx_index* idx, int64_t nprobe) {
    DFX_API_BEGIN
    idx->generation++;
    DFX_REQUIRE(nprobe >= 1, "nprobe must be >= 1");
    idx->nprobe = nprobe;
    DFX_API_END
}
int64_t dfx_get_nprobe(const dfx_index* idx) { return idx->nprobe; }
int64_t dfx_generation(const dfx_index* idx) { return (int64_t)idx->generation.load(); }
int64_t dfx_ntotal(const dfx_index* idx) { return idx->ntotal(); }
int64_t dfx_nlist(const dfx_index* idx) { return idx->is_flat() ? 0 : idx->cfg.nlist; }
int dfx_is_trained(const dfx_index* idx) { return (idx->trained || idx->flat_rows()) ? 1 : 0; }

int dfx_get_centroids(dfx_index* idx, float* out) {
    DFX_API_BEGIN
    DFX_REQUIRE(idx->is_ivf() && idx->trained, "index has no trained coarse quantizer");
    std::lock_guard<std::mutex> lk(idx->mu);
    DeviceGuard g(idx->cfg.device);
    idx->join_dev();
    DFX_CUDA(cudaMemcpy(out, idx->centroids.p, (size_t)idx->cfg.nlist * idx->cfg.d * 4, cudaMemcpyDeviceToHost));
    DFX_API_END
}

int dfx_merge_dev(int64_t S, int64_t nq, int64_t k, const float* d_D, const int64_t* d_I, int negate,
                  float* d_outD, int64_t* d_outI, void* stream) {
    DFX_API_BEGIN
    dfx_merge_impl(S, nq, k, d_D, d_I, negate, d_outD, d_outI, (cudaStream_t)stream);
    DFX_API_END
}
int dfx_merge(int64_t S, int64_t nq, int64_t k, const float* D, const int64_t* I, int negate, float* outD,
              int64_t* outI) {
    DFX_API_BEGIN
    int dev = 0;
    DFX_CUDA(cudaGetDevice(&dev));
    require_device(dev);
    if (nq <= 0) return 0;
    DevBuf dD, dI, oD, oI;
    size_t n = (size_t)S * nq * k;
    dD.reserve(n * 4);
    dI.reserve(n * 8);
    oD.reserve((size_t)nq * k * 4);
    oI.reserve((size_t)nq * k * 8);
    DFX_CUDA(cudaMemcpy(dD.p, D, n * 4, cudaMemcpyHostToDevice));
    DFX_CUDA(cudaMemcpy(dI.p, I, n * 8, cudaMemcpyHostToDevice));
    dfx_merge_impl(S, nq, k, dD.as<float>(), dI.as<int64_t>(), negate, oD.as<float>(), oI.as<int64_t>(), 0);
    DFX_CUDA(cudaMemcpy(outD, oD.p, (size_t)nq * k * 4, cudaMemcpyDeviceToHost));
    DFX_CUDA(cudaMemcpy(outI, oI.p, (size_t)nq * k * 8, cudaMemcpyDeviceToHost));
    DFX_API_END
}
int dfx_merge_packed_dev(int64_t R, int64_t S_loc, int64_t nq, int64_t k, const void* d_packed,
                         int64_t rank_stride_bytes, int64_t off_I_bytes, int negate, float* d_outD,
                         int64_t* d_outI, void* stream) {
    DFX_API_BEGIN
    dfx_merge_packed_impl(R, S_loc, nq, k, d_packed, rank_stride_bytes, off_I_bytes, negate, d_outD, d_outI,
                          (cudaStream_t)stream);
    DFX_API_END
}
int dfx_range_merge_dev(int64_t S, int64_t nq, const int64_t* d_lims, const float* d_D, const int64_t* d_P,
                        int64_t total, int maximize, int64_t* d_out_lims, float* d_outD, int64_t* d_outP,
                        int64_t* d_order, void* stream) {
    DFX_API_BEGIN
    dfx_range_merge_impl(S, nq, d_lims, d_D, d_P, total, maximize, d_out_lims, d_outD, d_outP, d_order,
                         (cudaStream_t)stream);
    DFX_API_END
}
int dfx_encode_ids_dev(int64_t n, const int64_t* d_ids, int64_t shard_tag, const int32_t* d_col,
                       int32_t drop_code, int64_t* d_out, void* stream) {
    DFX_API_BEGIN
    dfx_encode_ids_impl(n, d_ids, shard_tag, d_col, drop_code, d_out, (cudaStream_t)stream);
    DFX_API_END
}
int dfx_filter_compact_dev(int64_t nq, int64_t k_in, int64_t k_out, const float* d_D, const int64_t* d_I,
                           float* d_outD, int64_t* d_outI, int32_t* d_count, void* stream) {
    DFX_API_BEGIN
    dfx_filter_compact_impl(nq, k_in, k_out, d_D, d_I, d_outD, d_outI, d_count, (cudaStream_t)stream);
    DFX_API_END
}
int dfx_map_ids_dev(int64_t n, const int64_t* d_ids, const int64_t* d_table, int64_t* d_out, void* stream) {
    DFX_API_BEGIN
    dfx_map_ids_impl(n, d_ids, d_table, d_out, (cudaStream_t)stream);
    DFX_API_END
}

int dfx_last_stats(dfx_index* idx, int64_t* ndis, int64_t* nq, int64_t* nprobe) {
    DFX_API_BEGIN
    std::lock_guard<std::mutex> lk(idx->mu);
    DeviceGuard g(idx->cfg.device);
    idx->join_dev();
    int64_t nd = 0;
    dfx_stats_impl(idx, &nd, idx->stream);
    if (ndis) *ndis = nd;
    if (nq) *nq = idx->last_nq;
    if (nprobe) *nprobe = idx->last_nprobe;
    DFX_API_END
}

int dfx_profile_enable(dfx_index* idx, int on) {
    DFX_API_BEGIN
    std::lock_guard<std::mutex> lk(idx->mu);
    idx->prof_on = on != 0;
    DFX_API_END
}
int dfx_profile_read(dfx_index* idx, double* scan_ms, int64_t* scan_launches, int reset) {
    DFX_API_BEGIN
    std::lock_guard<std::mutex> lk(idx->mu);
    DeviceGuard g(idx->cfg.device);
    idx->join_dev();
    const double ms = idx->prof_scan.sum_ms();
    if (scan_ms) *scan_ms = ms;
    if (scan_launches) *scan_launches = (int64_t)idx->prof_scan.used;
    if (reset) {
        idx->prof_scan.reset();
        idx->prof_refine.reset();
    }
    DFX_API_END
}

// ------------------------------------------------------------------ state exchange
// How an array travels between the host and its device buffer: as it is, or converted on the host
// (ids: int64 exchanged, int32 stored; 4-bit codes: one per byte exchanged, two per byte stored)
enum class ExchangeConv { none, ids32, codes4 };

struct ExchangeArray {
    const char* name;
    DevBuf* buf;
    ExchangeConv conv;
    int64_t bytes;        // exchange size; a converted array is stored in bytes / 2
    bool needs_trained;   // dfx_get_array has it only once the index is trained
    bool importable;      // dfx_set_array accepts it
    const char* size_error;
};

// The arrays of the exchange format (include/dfx.h) that this index has, in import order, sized for
// the n_sorted vectors of the list-sorted storage
static std::vector<ExchangeArray> exchange_arrays(dfx_index* idx) {
    using C = ExchangeConv;
    const int kind = idx->cfg.kind;
    const int64_t n = idx->n_sorted, nlist = idx->cfg.nlist, d = idx->cfg.d, M = idx->M, M2 = idx->M2;
    if (kind == DFX_FLAT) return {{"xb", &idx->payload, C::none, n * d * 4, false, true, "xb: wrong size"}};
    if (kind == DFX_FLAT_SQ16)
        return {{"codes16", &idx->payload, C::none, n * d * 2, false, true, "codes16: wrong size (u16[ntotal, d])"}};
    if (kind == DFX_FLAT_PQ)
        return {{"codebooks", &idx->codebooks, C::none, M * idx->ksub * idx->dsub * 4, true, true, "codebooks: wrong size"},
                {"codes", &idx->payload, C::none, n * M, false, true, "codes: wrong size (u8[ntotal, M])"}};
    std::vector<ExchangeArray> a{{"centroids", &idx->centroids, C::none, nlist * d * 4, true, true, "centroids: wrong size"}};
    if (idx->has_pq())
        a.push_back({"codebooks", &idx->codebooks, C::none, M * idx->ksub * idx->dsub * 4, true, true, "codebooks: wrong size"});
    if (kind == DFX_IVF_SQ8)
        a.push_back({"sq_trained", &idx->sq_trained, C::none, 2 * d * 4, true, true,
                     "sq_trained: wrong size (2 * d floats: vmin, then vdiff)"});
    if (kind == DFX_IVF_PQR)
        a.push_back({"refine_codebooks", &idx->refine_cb, C::none, M2 * 256 * idx->dsub2 * 4, true, true,
                     "refine_codebooks: wrong size"});
    a.push_back({"list_off", &idx->list_off, C::none, (nlist + 1) * 8, true, true, "list_off: wrong size"});
    a.push_back({"ids", &idx->ids, C::ids32, n * 8, false, true, "ids: wrong size (set list_off first)"});
    if (idx->has_pq() && idx->ksub == 16)
        a.push_back({"codes", &idx->payload, C::codes4, n * M, false, true,
                     "codes: wrong size (one byte per code, u8[ntotal, M]; set list_off first)"});
    else
        a.push_back({kind == DFX_IVF_FLAT ? "vecs" : kind == DFX_IVF_SQ16 ? "codes16" : kind == DFX_IVF_SQ8 ? "codes8" : "codes",
                     &idx->payload, C::none, n * (int64_t)idx->row_bytes(), false, true,
                     "payload: wrong size (set list_off first)"});
    if (idx->pq_res()) a.push_back({"tvals", &idx->tvals, C::none, n * 4, false, false, nullptr});  // recomputed on import
    if (kind == DFX_IVF_PQR)
        a.push_back({"refine_codes", &idx->refine_codes, C::none, n * M2, false, true,
                     "refine_codes: wrong size (u8[ntotal, M2] in id order; set list_off first)"});
    if (idx->rflat())
        a.push_back({"refine_vecs", &idx->refine_vecs, C::none, n * d * 4, false, true,
                     "refine_vecs: wrong size (f32[ntotal, d] in id order; set list_off first)"});
    return a;
}

static const ExchangeArray* find_exchange_array(const std::vector<ExchangeArray>& arrays, const std::string& n) {
    for (const ExchangeArray& a : arrays)
        if (n == a.name) return &a;
    return nullptr;
}

int dfx_get_array(dfx_index* idx, const char* name, void* out, int64_t max_bytes, int64_t* nbytes) {
    DFX_API_BEGIN
    std::lock_guard<std::mutex> lk(idx->mu);
    DeviceGuard g(idx->cfg.device);
    idx->join_dev();
    if (idx->n_pending > 0) dfx_finalize_impl(idx, idx->stream);
    std::string n(name);
    struct Restore {  // the exchange format is row-major; put the interleaved form back afterwards
        dfx_index* i;
        bool on;
        ~Restore() {
            if (on) {
                try {
                    dfx_pq_rm_to_il(i, i->stream);
                } catch (...) {
                }
            }
        }
    } restore{idx, false};
    if (idx->il && (n == "codes" || n == "tvals" || n == "ids")) {
        dfx_pq_il_to_rm(idx, idx->stream);
        restore.on = true;
    }
    const std::vector<ExchangeArray> arrays = exchange_arrays(idx);
    const ExchangeArray* a = find_exchange_array(arrays, n);
    if (!a || (a->needs_trained && !idx->trained)) throw DfxError{"no array named '" + n + "' in this index"};
    const int64_t bytes = a->bytes;
    if (nbytes) *nbytes = bytes;
    if (!out) return 0;
    DFX_REQUIRE(max_bytes >= bytes, "output buffer too small for '" + n + "'");
    if (bytes == 0) return 0;
    if (a->conv == ExchangeConv::ids32) {
        std::vector<int32_t> tmp((size_t)bytes / 8);
        DFX_CUDA(cudaMemcpy(tmp.data(), a->buf->p, (size_t)bytes / 2, cudaMemcpyDeviceToHost));
        std::copy(tmp.begin(), tmp.end(), (int64_t*)out);
    } else if (a->conv == ExchangeConv::codes4) {
        std::vector<uint8_t> packed((size_t)bytes / 2);
        DFX_CUDA(cudaMemcpy(packed.data(), a->buf->p, packed.size(), cudaMemcpyDeviceToHost));
        uint8_t* o = (uint8_t*)out;
        for (size_t b = 0; b < packed.size(); b++) {  // M is even: byte b holds codes 2b and 2b + 1
            o[2 * b] = packed[b] & 15;
            o[2 * b + 1] = packed[b] >> 4;
        }
    } else {
        DFX_CUDA(cudaMemcpy(out, a->buf->p, (size_t)bytes, cudaMemcpyDeviceToHost));
    }
    DFX_API_END
}

int dfx_set_array(dfx_index* idx, const char* name, const void* in, int64_t nbytes) {
    DFX_API_BEGIN
    idx->generation++;
    std::lock_guard<std::mutex> lk(idx->mu);
    DeviceGuard g(idx->cfg.device);
    idx->join_dev();
    std::string n(name);
    if (idx->il) dfx_pq_il_to_rm(idx, idx->stream);  // imports arrive row-major
    const int64_t nlist = idx->cfg.nlist, d = idx->cfg.d;
    const std::vector<ExchangeArray> arrays = exchange_arrays(idx);
    const ExchangeArray* a = find_exchange_array(arrays, n);
    if (!a || !a->importable) throw DfxError{"cannot import array '" + n + "'"};
    if (idx->is_flat() && a->buf == &idx->payload) {  // the import of the rows sets their number
        const int64_t rb = (int64_t)idx->row_bytes();
        DFX_REQUIRE(nbytes % rb == 0, a->size_error);
        idx->n_sorted = nbytes / rb;
        idx->tc_flat_rows = -1;  // imported rows: any screening table is stale
    } else {
        DFX_REQUIRE(nbytes == a->bytes, a->size_error);
    }
    // the host conversions, which check the values they convert before anything is uploaded
    const void* src = in;
    int64_t dev_bytes = nbytes;
    std::vector<int32_t> ids32;
    std::vector<uint8_t> packed;
    if (a->conv == ExchangeConv::ids32) {
        const int64_t* s = (const int64_t*)in;
        ids32.resize((size_t)idx->n_sorted);
        for (int64_t i = 0; i < idx->n_sorted; i++) {
            DFX_REQUIRE(s[i] >= 0 && s[i] < (1ll << 31), "ids must be in [0, 2^31)");
            ids32[(size_t)i] = (int32_t)s[i];
        }
        if (idx->cfg.kind == DFX_IVF_PQR || idx->rflat()) {
            // the refine codes / rows are addressed by id (faiss asserts the same of IndexIVFPQR)
            std::vector<char> seen((size_t)idx->n_sorted, 0);
            for (int64_t i = 0; i < idx->n_sorted; i++) {
                DFX_REQUIRE(s[i] < idx->n_sorted && !seen[(size_t)s[i]],
                            std::string("ids: ") + (idx->rflat() ? "a flat refinement" : "an IVF-PQR index") +
                                " needs ids that are a permutation of 0 .. ntotal-1");
                seen[(size_t)s[i]] = 1;
            }
        }
        src = ids32.data();
        dev_bytes = nbytes / 2;
    } else if (a->conv == ExchangeConv::codes4) {
        const uint8_t* s = (const uint8_t*)in;
        packed.resize((size_t)nbytes / 2);
        for (size_t b = 0; b < packed.size(); b++) {
            DFX_REQUIRE(s[2 * b] < 16 && s[2 * b + 1] < 16, "codes: a 4-bit code must be in [0, 16)");
            packed[b] = (uint8_t)(s[2 * b] | (s[2 * b + 1] << 4));
        }
        src = packed.data();
        dev_bytes = nbytes / 2;
    }
    a->buf->reserve((size_t)std::max<int64_t>(dev_bytes, 4));
    if (dev_bytes) DFX_CUDA(cudaMemcpy(a->buf->p, src, (size_t)dev_bytes, cudaMemcpyHostToDevice));
    // what the uploaded array determines
    if (n == "centroids") {
        idx->cnorm.reserve((size_t)nlist * 4);
        dfx_launch_row_norms(idx->centroids.as<float>(), nlist, (int)d, idx->cnorm.as<float>(), idx->stream);
        DFX_CUDA(cudaStreamSynchronize(idx->stream));
    } else if (n == "codebooks") {
        idx->cbT_valid = false;
    } else if (n == "list_off") {
        idx->h_list_off.assign((const int64_t*)in, (const int64_t*)in + nlist + 1);
        DFX_REQUIRE(idx->h_list_off[0] == 0, "list_off[0] must be 0");
        idx->update_list_lengths();
        idx->n_sorted = idx->h_list_off[(size_t)nlist];
        idx->n_pending = 0;
    } else if (idx->flat_rows() && idx->cfg.metric == DFX_METRIC_L2) {  // "xb" / "codes16": the rows' norms
        idx->xnorm.reserve((size_t)std::max<int64_t>(idx->n_sorted, 1) * 4);
        dfx_with_flat_rows(idx, [&](auto rows) {
            dfx_launch_row_norms(rows, idx->n_sorted, (int)d, idx->xnorm.as<float>(), idx->stream);
        });
        DFX_CUDA(cudaStreamSynchronize(idx->stream));
    } else if (n == "refine_codes" || n == "refine_vecs") {
        idx->refine_cap = idx->refine_rows = idx->n_sorted;
    }
    idx->inv_valid = false;
    DFX_API_END
}

int dfx_import_done(dfx_index* idx) {
    DFX_API_BEGIN
    idx->generation++;
    std::lock_guard<std::mutex> lk(idx->mu);
    DeviceGuard g(idx->cfg.device);
    idx->join_dev();
    if (idx->is_ivf()) {
        DFX_REQUIRE(idx->centroids.p && idx->list_off.p, "import: centroids and list_off are required");
        if (idx->cfg.kind == DFX_IVF_PQR) {
            DFX_REQUIRE(idx->refine_cb.p, "import: refine_codebooks are required");
            DFX_REQUIRE(idx->refine_rows == idx->n_sorted, "import: refine_codes of every vector are required");
        }
        if (idx->rflat())
            DFX_REQUIRE(idx->refine_rows == idx->n_sorted, "import: refine_vecs of every vector are required");
        if (idx->pq_res()) {
            DFX_REQUIRE(idx->codebooks.p, "import: codebooks are required");
            dfx_compute_tvals_sorted(idx, idx->stream);  // K7 recomputes the per-vector term
            dfx_pq_rm_to_il(idx, idx->stream);
        }
        if (idx->cfg.kind == DFX_IVF_PQR) dfx_refresh_inv(idx, idx->stream);
        if (idx->cfg.kind == DFX_IVF_PQ_FS) DFX_REQUIRE(idx->codebooks.p, "import: codebooks are required");
        if (idx->cfg.kind == DFX_IVF_SQ8) DFX_REQUIRE(idx->sq_trained.p, "import: sq_trained is required");
        dfx_tc_prepare_centroids(idx, idx->stream);
        DFX_CUDA(cudaStreamSynchronize(idx->stream));
    }
    if (idx->cfg.kind == DFX_FLAT_PQ) DFX_REQUIRE(idx->codebooks.p, "import: codebooks are required");
    idx->trained = true;
    DFX_API_END
}

int dfx_free(void* p) {
    DFX_API_BEGIN
    if (p) DFX_CUDA(cudaFree(p));
    DFX_API_END
}

}  // extern "C"

// =====================================================================================
// synthetic data (bench harness).  Stateless: every value is a hash of (seed, stream, row, j).
// =====================================================================================
__host__ __device__ static inline uint64_t mix64(uint64_t z) {
    z = (z ^ (z >> 30)) * 0xbf58476d1ce4e5b9ull;
    z = (z ^ (z >> 27)) * 0x94d049bb133111ebull;
    return z ^ (z >> 31);
}
__host__ __device__ static inline uint64_t hash4(uint64_t seed, uint64_t stream, uint64_t a, uint64_t b) {
    uint64_t h = mix64(seed + 0x9e3779b97f4a7c15ull);
    h = mix64(h ^ (stream * 0xd1342543de82ef95ull + 0x632be59bd9b4e019ull));
    h = mix64(h ^ (a * 0x9e3779b97f4a7c15ull));
    h = mix64(h ^ (b * 0xc2b2ae3d27d4eb4full + 0x165667b19e3779f9ull));
    return h;
}
// standard normal from one 64-bit hash (Box-Muller on two 32-bit halves)
__device__ static inline float hash_normal(uint64_t h) {
    float u1 = ((float)(uint32_t)(h >> 32) + 0.5f) * (1.0f / 4294967296.0f);
    float u2 = ((float)(uint32_t)h + 0.5f) * (1.0f / 4294967296.0f);
    return sqrtf(-2.0f * __logf(u1)) * __cosf(6.28318530718f * u2);
}

// one CTA (128 threads) per row, d <= 4096, r <= 64
__global__ void synth_rows_kernel(dfx_synth p, const float* __restrict__ A, int64_t row0,
                                  const int64_t* __restrict__ rows, int64_t n, uint64_t noise_stream,
                                  float* __restrict__ out) {
    __shared__ float s_z[64];
    const int64_t r = blockIdx.x;
    if (r >= n) return;
    const int64_t row = rows ? rows[r] : row0 + r;
    const uint64_t cluster = (uint64_t)(row % p.nclusters);
    const uint64_t zkey = p.ngroups > 0 ? (uint64_t)(row % p.ngroups) : (uint64_t)row;
    if (threadIdx.x < p.r) {
        float z = hash_normal(hash4(p.seed, 2, zkey, threadIdx.x));
        z = p.sigma * fminf(4.f, fmaxf(-4.f, z));
        if (p.delta > 0.f) z += p.delta * hash_normal(hash4(p.seed, 5, (uint64_t)row, threadIdx.x));
        s_z[threadIdx.x] = z;
    }
    __syncthreads();
    for (int k = threadIdx.x; k < p.d; k += blockDim.x) {
        float mu = hash_normal(hash4(p.seed, 1, cluster, k));
        float az = 0.f;
        for (int j = 0; j < p.r; j++) az += A[k * p.r + j] * s_z[j];
        float v = mu + az;
        if (p.eps > 0.f) v += p.eps * hash_normal(hash4(p.seed, 4, (uint64_t)row, k));
        if (p.sigma_q > 0.f && noise_stream)
            v += p.sigma_q * hash_normal(hash4(p.seed, noise_stream, (uint64_t)row, k));
        out[r * p.d + k] = v;
    }
}

extern "C" {

// A: d x r with orthonormal columns (Gram-Schmidt of a hashed Gaussian matrix, on the host)
int dfx_synth_init(const dfx_synth* p, float** d_A_out, void* stream) {
    DFX_API_BEGIN
    DFX_REQUIRE(p && d_A_out, "null argument");
    DFX_REQUIRE(p->r >= 1 && p->r <= 64 && p->r <= p->d && p->d <= 4096, "synth: need 1 <= r <= min(64, d)");
    const int d = p->d, r = p->r;
    std::vector<double> A((size_t)d * r);
    for (int k = 0; k < d; k++)
        for (int j = 0; j < r; j++) {
            uint64_t h = hash4(p->seed, 3, (uint64_t)k, (uint64_t)j);
            double u1 = ((double)(uint32_t)(h >> 32) + 0.5) / 4294967296.0;
            double u2 = ((double)(uint32_t)h + 0.5) / 4294967296.0;
            A[(size_t)k * r + j] = std::sqrt(-2.0 * std::log(u1)) * std::cos(6.283185307179586 * u2);
        }
    for (int j = 0; j < r; j++) {
        for (int j2 = 0; j2 < j; j2++) {
            double dot = 0;
            for (int k = 0; k < d; k++) dot += A[(size_t)k * r + j] * A[(size_t)k * r + j2];
            for (int k = 0; k < d; k++) A[(size_t)k * r + j] -= dot * A[(size_t)k * r + j2];
        }
        double nrm = 0;
        for (int k = 0; k < d; k++) nrm += A[(size_t)k * r + j] * A[(size_t)k * r + j];
        nrm = std::sqrt(nrm);
        for (int k = 0; k < d; k++) A[(size_t)k * r + j] /= nrm;
    }
    std::vector<float> Af(A.begin(), A.end());
    float* dA = nullptr;
    DFX_CUDA(cudaMalloc(&dA, Af.size() * 4));
    DFX_CUDA(cudaMemcpyAsync(dA, Af.data(), Af.size() * 4, cudaMemcpyHostToDevice, (cudaStream_t)stream));
    DFX_CUDA(cudaStreamSynchronize((cudaStream_t)stream));
    *d_A_out = dA;
    DFX_API_END
}

int dfx_synth_rows_dev(const dfx_synth* p, const float* d_A, int64_t row0, const int64_t* d_rows, int64_t n,
                       uint64_t noise_stream, float* d_out, void* stream) {
    DFX_API_BEGIN
    if (n <= 0) return 0;
    DFX_REQUIRE(p->nclusters >= 1, "synth: nclusters >= 1");
    DFX_REQUIRE(p->ngroups == 0 || p->ngroups % p->nclusters == 0, "synth: ngroups must be a multiple of nclusters");
    DFX_LAUNCH(synth_rows_kernel, (unsigned)n, 128, 0, (cudaStream_t)stream, *p, d_A, row0, d_rows, n,
               noise_stream, d_out);
    DFX_API_END
}

}  // extern "C"
