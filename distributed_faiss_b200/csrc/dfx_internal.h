// dfx_internal.h -- index object + launcher declarations shared by the .cu files.
#pragma once
#include "dfx_common.cuh"
#include <vector>
#include <atomic>
#include <mutex>
#include <memory>
#include <algorithm>
#include <utility>
#include <type_traits>

// streaming multiprocessors of the current device (launch shapes are sized in waves over them)
int dfx_num_sms();
// dynamic shared memory one CTA of the current device may opt in to (bytes)
int dfx_smem_optin();

// A screening table of the tensor-core coarse quantizer (dfx_tc.cu): an index's centroids, the
// rows of a FLAT index, or the centroids of one k-means step.  Rows are screened centred on
// their mean m, which leaves the ranking unchanged and shrinks the screening error.
// The rows of a FLAT_SQ16 index are screened as they are stored: one exact fp16 plane (`rows`, the
// index's codes), no mean (m = 0, a zero vector in `mean`), scale 1, and the column term read
// from `rows_cterm` (L2: the stored |x|^2, IP: none) -- nothing per row is copied.
struct dfx_tc_table {
    DevBuf planes;        // fp16 [2][n_pad][d]: hi and lo planes of (c - m) * scale
    DevBuf cterm;         // f32 [n_pad]: column term, L2 |c - m|^2, IP -m.c; 3e38 for padded rows
    DevBuf mean;          // f32 [d] m, then f32 [2] and f64 [MEAN_CHUNKS][d] of work space
    float scale = 1.f;    // power of two of the planes
    float cmax2 = 0.f;    // max |c|^2
    float cmax2c = 0.f;   // max |c - m|^2
    const __half* rows = nullptr;        // one exact plane [n][d] (FLAT_SQ16), else nullptr
    const float* rows_cterm = nullptr;   // its column terms [n] (nullptr: 0), columns >= n never selected
    bool one_plane() const { return rows != nullptr; }
};

// Device time of one search stage (dfx_profile_enable): begin / end bracket its launches on a stream,
// sum_ms adds up the ranges since the last reset.  Event pairs are created on first use, then reused.
struct dfx_event_ranges {
    std::vector<std::pair<cudaEvent_t, cudaEvent_t>> ev;
    size_t used = 0;
    void begin(cudaStream_t st) {
        if (used == ev.size()) {
            cudaEvent_t a, b;
            DFX_CUDA(cudaEventCreate(&a));
            DFX_CUDA(cudaEventCreate(&b));
            ev.emplace_back(a, b);
        }
        DFX_CUDA(cudaEventRecord(ev[used++].first, st));
    }
    void end(cudaStream_t st) { DFX_CUDA(cudaEventRecord(ev[used - 1].second, st)); }
    double sum_ms() {  // synchronises
        double ms = 0;
        for (size_t i = 0; i < used; i++) {
            DFX_CUDA(cudaEventSynchronize(ev[i].second));
            float t = 0;
            DFX_CUDA(cudaEventElapsedTime(&t, ev[i].first, ev[i].second));
            ms += t;
        }
        return ms;
    }
    void reset() { used = 0; }
    void destroy() {
        for (auto& e : ev) {
            cudaEventDestroy(e.first);
            cudaEventDestroy(e.second);
        }
    }
};

// A runtime value as a template argument: calls f(std::integral_constant<int, V>{}) for the V of
// the list that equals v, and returns false when none does.  Every V of the list is instantiated.
template <int... Vs> using IntList = std::integer_sequence<int, Vs...>;
template <int... Vs, class F>
static bool dispatch_int(IntList<Vs...>, int v, F&& f) {
    return ((v == Vs && (f(std::integral_constant<int, Vs>{}), true)) || ...);
}

struct dfx_index {
    dfx_cfg cfg{};
    int M = 0, ksub = 0, dsub = 0;
    int64_t nprobe = 1;  // faiss default (index.py:47 copies it back into cfg for knnlm)
    bool trained = false;

    // list-sorted storage ("sorted") and arrival-order staging ("pending")
    int64_t n_sorted = 0, n_pending = 0;
    DevBuf centroids, cnorm, codebooks;
    DevBuf sq_trained;                  // IVF_SQ8: f32[2][d] = vmin, vdiff (faiss ScalarQuantizer::trained)
    DevBuf list_off;                    // int64[nlist+1]
    std::vector<int64_t> h_list_off;    // host mirror
    // h_len_top[p]: vectors in the p longest lists together (bounds one query's candidates at k > 1024)
    std::vector<int64_t> h_len_top;
    DevBuf ids;                         // int32[n_sorted] shard-local ids, list-sorted
    DevBuf payload;                     // kind-specific rows, list-sorted (FLAT, FLAT_SQ16, FLAT_PQ: arrival order)
    DevBuf tvals;                       // IVF_PQ: f32[n_sorted] (IVF_PQ_FS has none)
    DevBuf xnorm;                       // FLAT / FLAT_SQ16 + L2: f32[n], |x|^2 of the stored rows
    DevBuf p_list, p_payload, p_tvals;  // pending: int32 list per row, payload rows, tvals
    int64_t p_cap = 0;
    int64_t reserve_hint = 0;

    // search workspace (grow-only)
    DevBuf w_vals, w_keys, w_dis0, w_lut, w_part, w_q, w_D, w_I, w_misc, w_best;
    DevBuf w_coff;  // k > 1024: int64 [qc][nprobe + 1] slot offsets of the candidate rows (in w_part)
    // reconstruct support: inverse of ids (shard-local id -> storage position)
    DevBuf inv;
    bool inv_valid = false;
    // training knobs (dfx_set_param)
    int kmeans_niter = 25;            // faiss Clustering default niter
    int max_points_per_centroid = 256;  // faiss Clustering default
    uint64_t train_seed = 1234;       // faiss Clustering default seed

    // IVF-PQ, M == 32: block-interleaved storage for the lane-per-vector scan (dfx_scan_il2.cu,
    // layout dfx_il2_byte).  While `il` is set the row-major payload/tvals/ids are released.
    bool il = false, il_enabled = true;
    DevBuf il_codes, il_tvals, il_ids, blk_off;
    int64_t nblk = 0;
    DevBuf codebooksT;  // [ksub][M][dsub]: the order the fused table build reads (dfx_scan_il2.cu)
    bool cbT_valid = false;

    // tensor-core coarse quantizer (dfx_tc.cu): the index's screening table, the one of a k-means
    // step, and screening workspace (tc_qn: f32x2 (|q|^2, |q - m|^2) per query row, tc_qterm its row term)
    dfx_tc_table tc_tab, tc_tab_tmp;
    DevBuf tc_q, tc_qmult, tc_qterm, tc_gmin, tc_tmin, tc_gmin2, tc_gargc, tc_groups, tc_cand, tc_qn, tc_amb, tc_ovf;
    // screening precision (dfx_tc.cu): tc_mode 0 = AUTO, 1 = FAST (one fp16 MMA per k-step),
    // 2 = PRECISE (hi/lo split, three MMAs).  AUTO starts PRECISE and moves to FAST once a launch
    // shows that FAST's wider tolerance would not overflow the kept groups (and back if it does).
    int tc_mode = 0;
    bool tc_fast = false;       // the precision the next screening launch uses (AUTO state)
    int32_t* tc_stat_h = nullptr;      // pinned [2]: {overflow rows, rows that FAST would overflow} of a past launch
    cudaEvent_t tc_stat_ev = nullptr;
    bool tc_stat_pending = false, tc_stat_fast = false;
    int64_t tc_stat_rows = 0;
    int64_t tc_last_rows = 0, tc_last_overflow = 0, tc_last_fast_would = 0;  // of the last launch polled
    int64_t tc_auto_window = 16384;            // AUTO: rows observed before PRECISE may become FAST
    int64_t tc_acc_rows = 0, tc_acc_bad = 0;   // AUTO: rows / rows that (would) overflow since the last decision
    bool tc_ready = false;
    bool tc_enabled = true;
    int rows_inflight = 0;      // vectors in flight per warp of scan_rows_kernel: 0 = by row size, else 4 / 8
    int il2_threads = 0;        // scan_pq_il2 CTA shape: 0 = default (env DFX_IL2_THREADS or 256), 256, 512
    int il2_prefetch = -1;      // L2 prefetch distance in blocks: -1 = default (env DFX_IL2_PREFETCH or 4)
    bool flat_tc = true;        // FLAT / FLAT_SQ16: search through the tensor-core screening (dfx_tc_flat_candidates)
    int64_t tc_flat_rows = -1;  // rows covered by the screening table of a flat index (-1: none)
    bool tc_flat_finite = true; // FLAT_SQ16: every code of those rows is finite (else the FFMA GEMM serves)

    // IVF_PQR: the refinement PQ (M2 sub-quantizers of 256 centroids, dsub2 = d / M2), its codes by
    // id (u8[ntotal][M2], arrival order; refine_cap rows allocated), k' = k * k_factor, and the
    // per-chunk workspace of the re-ranking (first-stage D' / I' and the refined composites)
    int M2 = 0, dsub2 = 0;
    float k_factor = 4.f;  // faiss IndexIVFPQR default
    DevBuf refine_cb, refine_codes;
    int64_t refine_cap = 0, refine_rows = 0;  // rows allocated / rows imported (dfx_set_array)
    DevBuf w_rD, w_rI, w_rcomp;
    // flat refinement (cfg.refine_flat): the raw rows by id (f32[ntotal][d], arrival order), sharing
    // refine_cap / refine_rows, k_factor (default 1, faiss IndexRefine) and the workspace above
    DevBuf refine_vecs;

    // profiling (dfx_profile_enable): each query chunk's table prep + list scan (dfx_profile_read),
    // and the re-ranking stage of IVF_PQR and the flat refinement (dfx_get_param "refine_ms")
    bool prof_on = false;
    dfx_event_ranges prof_scan, prof_refine;

    // last-search bookkeeping
    int64_t last_nq = 0, last_nprobe = 0;
    bool last_keys_valid = false;

    // range search (dfx_search.cu, "Range search"): the results of the last one, r_total composites
    // (r_comp) with their query (r_qidx), grouped by query and sorted; r_total = -1 when there are none
    // to fetch.  r_comp2 / r_qidx2 are the sorts' spare buffers, r_cnt / r_off a piece's per-query
    // counts and offsets, r_tot the per-query totals of the call, r_qn FLAT L2's |q|^2, r_lims the
    // host entry point's lims.
    DevBuf r_comp, r_qidx, r_comp2, r_qidx2, r_cnt, r_off, r_tot, r_tmp, r_qn, r_lims;
    int64_t r_total = -1;
    int r_metric = 0;
    bool r_qnorm = false;  // the mapping adds r_qn back (FLAT L2)

    // bumped by every call that can change what a search launches (train / add / finalize /
    // import / set_param / set_nprobe): CUDA-graph replays of a search are keyed on it
    std::atomic<long long> generation{0};

    cudaStream_t stream = nullptr;  // used by the host-pointer entry points
    // stream of the most recent *_dev call; host-pointer entry points (which run on `stream`,
    // a non-blocking stream) wait for it first so that the two never race
    cudaStream_t last_dev_stream = nullptr;
    bool dev_work_pending = false;
    // An EVENT after the call's own work, not the stream: the caller may queue unrelated work
    // behind it on the same stream -- the search plane queues the wait for the NEXT header
    // broadcast, which only completes when the client rank sends one, and a socket search served
    // meanwhile by another thread of the same process must not wait for that (it deadlocked the
    // 2-GPU bench: rank 0 waited for the socket reply, rank 1's reply for rank 0's next header).
    cudaEvent_t dev_done = nullptr;
    bool dev_done_recorded = false;
    void note_dev(cudaStream_t st) {
        last_dev_stream = st;
        dev_work_pending = true;
        dev_done_recorded = false;
        cudaStreamCaptureStatus cs = cudaStreamCaptureStatusNone;
        if (cudaStreamIsCapturing(st, &cs) != cudaSuccess) cudaGetLastError();
        if (cs != cudaStreamCaptureStatusNone) return;  // inside a graph capture: the capturing caller orders its replays
        if (!dev_done && cudaEventCreateWithFlags(&dev_done, cudaEventDisableTiming) != cudaSuccess) {
            cudaGetLastError();
            dev_done = nullptr;
        }
        if (dev_done && cudaEventRecord(dev_done, st) == cudaSuccess) dev_done_recorded = true;
        else cudaGetLastError();
    }
    // a *_dev call on a different stream than the previous one: order them
    void join_dev_if_other(cudaStream_t st) {
        if (dev_work_pending && st != last_dev_stream) join_dev();
    }
    void join_dev() {
        if (dev_work_pending) {
            if (dev_done_recorded) cudaEventSynchronize(dev_done);
            else cudaStreamSynchronize(last_dev_stream);
            dev_work_pending = false;
        }
    }
    std::mutex mu;

    size_t row_bytes() const {
        switch (cfg.kind) {
            case DFX_FLAT:
            case DFX_IVF_FLAT: return (size_t)cfg.d * 4;
            case DFX_FLAT_SQ16: return (size_t)cfg.d * 2;
            case DFX_FLAT_PQ: return (size_t)M;
            case DFX_IVF_PQ: return ksub == 16 ? (size_t)M / 2 : (size_t)M;  // 4-bit codes: two per byte
            case DFX_IVF_PQ_FS: return (size_t)M / 2;
            case DFX_IVF_PQR: return (size_t)M;  // the refine codes live outside the lists
            case DFX_IVF_SQ16: return (size_t)cfg.d * 2;
            case DFX_IVF_SQ8: return (size_t)cfg.d;
        }
        return 0;
    }
    int64_t ntotal() const { return n_sorted + n_pending; }
    // after every change of h_list_off
    void update_list_lengths() {
        const size_t nl = h_list_off.empty() ? 0 : h_list_off.size() - 1;
        std::vector<int64_t> len(nl);
        for (size_t l = 0; l < nl; l++) len[l] = h_list_off[l + 1] - h_list_off[l];
        std::sort(len.begin(), len.end(), [](int64_t a, int64_t b) { return a > b; });
        h_len_top.assign(nl + 1, 0);
        for (size_t l = 0; l < nl; l++) h_len_top[l + 1] = h_len_top[l] + len[l];
    }
    // the kinds without lists or probes: every stored row is scored by every search, rows are kept in
    // arrival order, and ids are positions (FLAT: fp32 rows, FLAT_SQ16: fp16 rows, FLAT_PQ: 8-bit PQ codes)
    bool is_flat() const { return cfg.kind == DFX_FLAT || cfg.kind == DFX_FLAT_SQ16 || cfg.kind == DFX_FLAT_PQ; }
    bool is_ivf() const { return !is_flat(); }
    // the flat kinds that store the rows themselves (FLAT, FLAT_SQ16): trained at creation, searched by the
    // GEMM or the tensor-core screening, with |x|^2 kept under L2.  FLAT_PQ is trained and scores codes.
    bool flat_rows() const { return cfg.kind == DFX_FLAT || cfg.kind == DFX_FLAT_SQ16; }
    bool rflat() const { return cfg.refine_flat != 0; }
    // the kinds with PQ codebooks (IVF_PQ / IVF_PQR: residual codes, IVF_PQ_FS and FLAT_PQ: codes of the
    // raw vectors)
    bool has_pq() const {
        return cfg.kind == DFX_IVF_PQ || cfg.kind == DFX_IVF_PQ_FS || cfg.kind == DFX_IVF_PQR || cfg.kind == DFX_FLAT_PQ;
    }
    // the kinds whose lists hold IVF-PQ residual codes with t-values (IVF_PQR: its first stage)
    bool pq_res() const { return cfg.kind == DFX_IVF_PQ || cfg.kind == DFX_IVF_PQR; }
};

// ---- dfx_search.cu
// values[q][j] = ranking value of row (col0+j) of X for query q (IP: -q.x ; L2: |x|^2 - 2 q.x)
void dfx_launch_gemm_values(const float* Q, int64_t nq, const float* X, const float* xnorm,
                            int64_t ncols, int d, int metric, float* out, int64_t ld_out,
                            cudaStream_t st);
void dfx_launch_gemm_values(const float* Q, int64_t nq, const __half* X, const float* xnorm,
                            int64_t ncols, int d, int metric, float* out, int64_t ld_out,
                            cudaStream_t st);
void dfx_launch_row_norms(const float* X, int64_t n, int d, float* out, cudaStream_t st);
void dfx_launch_row_norms(const __half* X, int64_t n, int d, float* out, cudaStream_t st);
// the stored rows of a flat index as their element type: f(const float*) for FLAT, f(const __half*)
// for FLAT_SQ16
template <class F>
static auto dfx_with_flat_rows(const dfx_index* idx, F&& f) {
    if (idx->cfg.kind == DFX_FLAT_SQ16) return f(idx->payload.as<__half>());
    return f(idx->payload.as<float>());
}
// top-k columns per row of a values matrix -> keys int32[nrows,k] (and optional values)
void dfx_launch_select_cols(const float* vals, int64_t nrows, int n, int64_t ld, int k,
                            uint32_t col_base, int32_t* keys, float* kvals, uint64_t* comp_out,
                            int64_t comp_ld, cudaStream_t st);
void dfx_search_impl(dfx_index* idx, int64_t nq, const float* d_x, int64_t k, float* d_D,
                     int64_t* d_I, cudaStream_t st);
void dfx_merge_impl(int64_t S, int64_t nq, int64_t k, const float* d_D, const int64_t* d_I,
                    int negate, float* d_outD, int64_t* d_outI, cudaStream_t st);
void dfx_merge_packed_impl(int64_t R, int64_t S_loc, int64_t nq, int64_t k, const void* d_packed,
                           int64_t rank_stride, int64_t off_I, int negate, float* d_outD,
                           int64_t* d_outI, cudaStream_t st);
void dfx_range_merge_impl(int64_t S, int64_t nq, const int64_t* d_lims, const float* d_D, const int64_t* d_P,
                          int64_t total, int maximize, int64_t* d_out_lims, float* d_outD, int64_t* d_outP,
                          int64_t* d_order, cudaStream_t st);
void dfx_encode_ids_impl(int64_t n, const int64_t* d_ids, int64_t tag, const int32_t* d_col,
                         int32_t drop_code, int64_t* d_out, cudaStream_t st);
void dfx_filter_compact_impl(int64_t nq, int64_t kin, int64_t kout, const float* d_D, const int64_t* d_I,
                             float* d_outD, int64_t* d_outI, int32_t* d_count, cudaStream_t st);
void dfx_map_ids_impl(int64_t n, const int64_t* d_ids, const int64_t* d_table, int64_t* d_out,
                      cudaStream_t st);
void dfx_stats_impl(dfx_index* idx, int64_t* ndis, cudaStream_t st);
// range search of nq device queries: d_lims int64[nq + 1] (device), *total = lims[nq] (host);
// synchronises once per piece and once at the end.  The results stay in r_comp / r_qidx until
// dfx_range_fetch_impl maps them to (D, I)
void dfx_range_impl(dfx_index* idx, int64_t nq, const float* d_x, float radius, int64_t* d_lims, int64_t* total,
                    cudaStream_t st);
void dfx_range_fetch_impl(dfx_index* idx, float* d_D, int64_t* d_I, cudaStream_t st);

void dfx_launch_select_comp(const uint64_t* comp, int64_t nrows, int n, int64_t ld, int k, int32_t* keys,
                            cudaStream_t st);

// Interleaved IVF-PQ block (M == 32): 32 vectors x 32 codes = 1 KB, one lane per vector.
// Lane v of the scanning warp owns vector v of
// the block and walks its 32 subquantizers in the rotated order m = (t + v) & 31, t = 0..31, so
// that at every step the 32 lanes read 32 different table columns (bank == column).  Byte t of
// the lane's 32 code bytes therefore holds the code of subquantizer (t + v) & 31; the two 16-byte
// halves of all lanes are stored contiguously (bytes 0..511: t = 0..15 of lanes 0..31, bytes
// 512..1023: t = 16..31) so that each of the two 128-bit loads of a warp is one 512-byte run.
__host__ __device__ __forceinline__ int dfx_il2_byte(int v, int m) {
    const int t = (m - v) & 31;
    return (t >> 4) * 512 + v * 16 + (t & 15);
}
// (the `layout` argument of the C-ABI probe dfx_debug_il_byte is kept for compatibility; there is
// one block layout)
__host__ __device__ __forceinline__ int dfx_il_byte_of(int /*layout*/, int v, int m) { return dfx_il2_byte(v, m); }

// ---- dfx_scan_il.cu
bool dfx_il_wanted(const dfx_index* idx);
void dfx_pq_rm_to_il(dfx_index* idx, cudaStream_t st);
void dfx_pq_il_to_rm(dfx_index* idx, cudaStream_t st);
// ---- dfx_scan_il2.cu: K3 + K4 fused; returns true when it wrote the final (D, I) rows itself
bool dfx_launch_scan_pq_il2(dfx_index* idx, const float* xq, int64_t qc, const int32_t* keys, int nprobe, int G,
                            int ngroups, int k, int cap, uint64_t* part, float* outD, int64_t* outI,
                            cudaStream_t st);
// k > 1024: the same scan writing every vector's composite to its slot of the candidate rows
void dfx_launch_scan_pq_il2_mat(dfx_index* idx, const float* xq, int64_t qc, const int32_t* keys, int nprobe, int G,
                                int ngroups, uint64_t* cand, const int64_t* coff, cudaStream_t st);

// ---- dfx_tc.cu
bool dfx_tc_supported(int d);
void dfx_tc_stats_sync(dfx_index* idx);  // wait for and fold in the statistics of the last screening launch
void dfx_tc_prepare_centroids(dfx_index* idx, cudaStream_t st);
void dfx_tc_coarse_search(dfx_index* idx, const float* d_x, int64_t nq, int nprobe, int32_t* keys,
                          cudaStream_t st);
// the flat searches dfx_tc_flat_candidates serves (d as dfx_tc_supported, N >= 1024, k <= 100)
bool dfx_tc_flat_covers(const dfx_index* idx, int k);
// (re)builds the screening table of a flat index's rows when they changed; false when the rows cannot
// be screened (a FLAT_SQ16 index holding a non-finite code), which leaves the search to the FFMA GEMM
bool dfx_tc_flat_table(dfx_index* idx, cudaStream_t st);
int dfx_tc_flat_candidates(dfx_index* idx, const float* d_x, int64_t nq, int k, cudaStream_t st);
void dfx_tc_debug_screen(dfx_index* idx, int64_t nq, const float* d_x, int npl, float* gmin, float* gmin2,
                         uint8_t* gargc, cudaStream_t st);
void dfx_tc_assign(dfx_index* idx, int d, const float* d_cent, const float* d_cnorm, int64_t nlist, int metric,
                   int64_t n, const float* d_x, int32_t* d_assign, cudaStream_t st);

// ---- dfx_build.cu
void dfx_train_impl(dfx_index* idx, int64_t n, const float* d_x, cudaStream_t st);
void dfx_add_impl(dfx_index* idx, int64_t n, const float* d_x, cudaStream_t st);
void dfx_finalize_impl(dfx_index* idx, cudaStream_t st);
// tag < 0: d_ids are shard-local ids (unknown / -1 rows become NaN); tag >= 0: d_ids are exchange
// ids and only the rows owned by shard `tag` are written
void dfx_reconstruct_impl(dfx_index* idx, int64_t n, const int64_t* d_ids, float* d_out,
                          cudaStream_t st, int64_t tag = -1);
// fused nearest-centroid (GEMM + argmin epilogue), no values matrix
void dfx_launch_assign_fused(const float* X, int64_t n, const float* cent, const float* cnorm,
                             int64_t nlist, int d, int metric, unsigned long long* best,
                             int32_t* out, cudaStream_t st);
void dfx_assign_impl(dfx_index* idx, const float* d_cent, const float* d_cnorm, int64_t nlist,
                     int metric, int d, int64_t n, const float* d_x, int32_t* d_assign,
                     cudaStream_t st);
void dfx_compute_tvals_sorted(dfx_index* idx, cudaStream_t st);
// `inv` (shard-local id -> storage position, padded block position when interleaved) for the
// current layout; a no-op while it is valid.  IVF_PQR searches read it, so every change of the
// layout rebuilds it right away (dfx_layout_changed; import).
void dfx_refresh_inv(dfx_index* idx, cudaStream_t st);
// after every change of the storage layout (train, finalize, the interleaved conversions): `inv` is
// stale, and an IVF_PQR shard rebuilds it at once, so a search captured into a CUDA graph depends on
// no host flag
void dfx_layout_changed(dfx_index* idx, cudaStream_t st);
