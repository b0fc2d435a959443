/*
 * dfx.h -- C-ABI of the H100-native shard engine (libdfx.so).
 *
 * This is the drop-in boundary for the SEARCH PATH of
 * facebookresearch/distributed-faiss.  The reference is pure Python and
 * reaches its numeric kernels through the SWIG-wrapped `faiss` object that
 * `distributed_faiss/index.py` keeps in `Index.faiss_index`; each entry point
 * below names the reference call site (file:line in the reference repository) whose
 * faiss call it replaces.  Plain pointers and sizes only -- no torch types.
 *
 * Conventions
 *   - every function returns 0 on success, non-zero on error; the message is
 *     available from dfx_last_error() (thread-local).  The Python binding
 *     turns it into RuntimeError, which IndexServer forwards to the client as
 *     rpc.ServerException exactly like a faiss exception (server.py:229-236).
 *   - "_dev" variants take DEVICE pointers and a cudaStream_t (passed as
 *     void*), enqueue work and return without synchronising; the others take
 *     HOST pointers, copy in/out and synchronise (the reference-facing path).
 *   - float32 row-major C-contiguous inputs, like faiss (index.py:151 casts,
 *     index.py:257 does not).
 *   - results follow faiss: L2 ascending / IP descending, missing entries
 *     id -1 and distance +FLT_MAX (L2) or -FLT_MAX (IP).  Ties are broken by
 *     the total order (value asc, id asc) -- see DESIGN.md.
 *   - there is no CPU fallback: every entry point that computes requires a
 *     CUDA device of compute capability 10.x and fails otherwise.
 */
#ifndef DFX_H
#define DFX_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct dfx_index dfx_index;

/* which faiss object the reference builder would have made (index.py:93-100) */
enum {
    DFX_FLAT = 0,     /* faiss.IndexFlatIP / IndexFlatL2         index.py:94, 25-33 */
    DFX_IVF_FLAT = 1, /* faiss.IndexIVFFlat                       index.py:36-40     */
    DFX_IVF_PQ = 2,   /* faiss.IndexIVFPQ (L2, by_residual)       index.py:43-48     */
    DFX_IVF_SQ16 = 3, /* faiss.IndexIVFScalarQuantizer(QT_fp16)   index.py:63-68     */
    DFX_IVF_SQ8 = 4,  /* faiss.IndexIVFScalarQuantizer(QT_8bit), by_residual: the factory string
                         "IVF{n},SQ8" (index.py:380-396) -- one byte per dimension */
    DFX_IVF_PQ_FS = 5, /* faiss.IndexIVFPQFastScan(nbits = 4), NOT by_residual: the factory string
                         "IVF{n},PQ{M}x4fs" (index.py:380-396).  4-bit codes packed two per byte; the
                         search quantizes each query's distance table to 8 bits and sums it in
                         integers (DESIGN.md section 2).  L2 only, for the index and its quantizer */
    DFX_IVF_PQR = 6,  /* faiss.IndexIVFPQR: the factory string "IVF{n},PQ{M}+{M2}" (index.py:380-396).
                         An 8-bit IVF-PQ (by_residual) whose residual error is encoded again by a second
                         8-bit PQ of M2 bytes, stored by id outside the lists.  A search runs the IVF-PQ
                         search for k' = k * k_factor candidates and re-ranks them on the reconstruction
                         c + PQ1 + PQ2 (DESIGN.md section 2).  L2 only, for the index and its quantizer */
    DFX_FLAT_SQ16 = 7, /* faiss.IndexScalarQuantizer(d, QT_fp16, metric): the factory string "SQfp16"
                         (index.py:385-396).  No training.  Each row is stored as its fp16 rounding
                         (2 d bytes per vector, plus its fp32 squared norm under L2), ids are positions,
                         and a search returns bit for bit what a FLAT index of the same metric returns over
                         the decoded rows (DESIGN.md section 2).  nlist, pq_m, pq_nbits, refine_m and
                         refine_flat must be 0 */
    DFX_FLAT_PQ = 8   /* faiss.IndexPQ(d, M, 8, metric): the factory string "PQ{M}" / "PQ{M}x8"
                         (index.py:385-396).  Trained (one 256-centroid k-means per sub-quantizer on the
                         raw sub-vectors), no lists: each row is stored as its M one-byte codes in arrival
                         order, ids are positions, and a search sums each query's [M][256] distance table
                         (L2, or the negated inner product) over the codes of every row (DESIGN.md
                         section 2).  nlist, refine_m and refine_flat must be 0 */
};

/* faiss.METRIC_INNER_PRODUCT / faiss.METRIC_L2 (index_cfg.py:44-52) */
enum { DFX_METRIC_IP = 0, DFX_METRIC_L2 = 1 };

typedef struct dfx_cfg {
    int32_t kind;     /* DFX_FLAT ... */
    int32_t metric;   /* FLAT / IVF_FLAT / FLAT_SQ16 / FLAT_PQ: search metric.  IVF_PQ / IVF_SQ16 / IVF_SQ8: metric of
                         the coarse quantizer only -- the reference never forwards it to the
                         index, which is therefore always L2 (index.py:44-46, 64-66).
                         IVF_PQ_FS: must be L2 (an inner-product metric is refused). */
    int32_t d;        /* vector dimension (cfg.dim) */
    int32_t pq_m;     /* IVF_PQ: sub-quantizers  (cfg.extra["code_size"], index.py:44).  8-bit codes
                         (and IVF_PQR): 4 <= M <= 128, M % 4 == 0, d % M == 0 (128: one query's fp32
                         table, M x 256 x 4 B, must fit in one thread block's shared memory).  4-bit
                         codes and IVF_PQ_FS: 8 <= M <= 128, M % 8 == 0, d % M == 0.  FLAT_PQ:
                         sub-quantizers, as for 8-bit IVF_PQ */
    int32_t pq_nbits; /* IVF_PQ: bits per code   (cfg.extra["bits_per_vector"], index.py:45): 8, or 4
                         (ksub = 16; codes stored two per byte, low nibble first, as faiss packs
                         them).  IVF_PQ_FS: must be 4.  IVF_PQR and FLAT_PQ: must be 8 */
    int32_t device;   /* CUDA device ordinal this shard lives on */
    int64_t nlist;    /* IVF_*: number of inverted lists (cfg.centroids); IVF kinds need d % 4 == 0.
                         Must be 0 for FLAT_SQ16 and FLAT_PQ */
    int32_t refine_m; /* IVF_PQR: sub-quantizers of the refinement PQ (M2; 8 bits each): 4 <= M2 <= 128,
                         M2 % 4 == 0, d % M2 == 0.  Must be 0 for every other kind */
    int32_t refine_flat; /* non-zero: flat refinement (faiss IndexRefineFlat, the ",RFlat" suffix of a
                         factory string) on top of IVF_PQ with 8-bit codes, IVF_PQ_FS, IVF_SQ8 or IVF_SQ16:
                         the raw fp32 rows are kept by id next to the lists ("refine_vecs", 4 d bytes per
                         vector), a search runs the base kind's search for k' = k * k_factor candidates
                         and re-ranks them on their exact L2 distances, and a reconstruction returns
                         the stored row.  The metric must be L2.  Must be 0 for FLAT, IVF_FLAT, IVF_PQR
                         and IVF_PQ with 4-bit codes */
} dfx_cfg;

/* ---- lifetime: replaces the faiss constructors at index.py:25-48,63-68,94 ---- */
int dfx_create(const dfx_cfg *cfg, dfx_index **out);
void dfx_destroy(dfx_index *idx);

/* ---- build: faiss_index.train(x) index.py:217 ; faiss_index.add(x) index.py:425 ---- */
int dfx_train(dfx_index *idx, int64_t n, const float *x);
int dfx_add(dfx_index *idx, int64_t n, const float *x);
int dfx_train_dev(dfx_index *idx, int64_t n, const float *d_x, void *stream);
int dfx_add_dev(dfx_index *idx, int64_t n, const float *d_x, void *stream);
/* knobs (every setting returns the same results; they only move the cost):
 * training: "kmeans_niter" (default 25), "max_points_per_centroid" (256), "train_seed" (1234) --
 *   the faiss Clustering defaults;
 * "tensor_cores" (1): 0 forces the plain fp32 FFMA coarse quantizer instead of the wgmma
 *   screening path;
 * "tc_screen_mode" (0): precision of the wgmma screening: 0 = AUTO (starts PRECISE, moves to
 *   FAST once enough rows have shown that FAST's wider tolerance would not overflow the kept
 *   groups, and back as soon as it does),
 *   1 = FAST (fp16 operands, one MMA per k-step), 2 = PRECISE (fp16 hi/lo split, three MMAs);
 *   "tc_auto_window" (16384): rows AUTO observes before PRECISE may become FAST;
 * "flat_tensor_cores" (1): 0 runs FLAT and FLAT_SQ16 searches through the FFMA GEMM instead of the
 *   tensor-core screening + exact re-rank (a FLAT_SQ16 shard holding a non-finite code, an input
 *   beyond +-65504, always takes the FFMA GEMM);
 * "interleaved" (1): 0 keeps IVF-PQ (M = 32) codes row-major (one vector per lane, table from
 *   pq_prep_kernel) instead of the block-interleaved layout of the fused table-build + scan;
 * "il2_threads" (0 = 256) / "il2_prefetch" (-1 = 4 blocks): CTA shape and L2 prefetch distance of
 *   that scan (tuning; 512 threads at k > 512 do not fit in shared memory and run with 256);
 * "rows_inflight" (0 = by row size): 4 or 8 vectors per warp in flight in the IVF-Flat / IVF-SQ
 *   list scan;
 * "k_factor" (IVF_PQR: 4; refine_flat: 1 -- the faiss defaults of IndexIVFPQR and IndexRefine; no
 *   other index has it; this knob DOES change results): a search for k results re-ranks the
 *   k' = (int64)((float)k * k_factor) best candidates of the first stage, as faiss's k_factor;
 *   values outside [1, 16384] are refused, and a search whose k' exceeds 16384 raises before
 *   launching anything */
int dfx_set_param(dfx_index *idx, const char *name, double value);
/* read back a knob or a counter: the names of dfx_set_param, plus "tc_fast" (the precision the
 * next screening launch will use: 1 = FAST), "tc_stat_rows" / "tc_stat_overflow" /
 * "tc_stat_fast_would" (rows, rows re-done exactly, and rows FAST would have re-done, of the last
 * launch whose statistics came back; synchronises with that launch), "workspace_bytes" (bytes of
 * the partial-result workspace, the largest any search so far has needed, including the candidate
 * rows of IVF searches with k > 1024; IVF searches keep it within 128 MiB by their query chunk),
 * "refine_ms" / "refine_launches" (IVF_PQR / refine_flat with profiling on: summed device time and number of
 * the refinement stages -- re-rank kernel and final selection -- since the last reset of
 * dfx_profile_read; synchronises), "index_bytes" (bytes of device memory the index's persistent
 * arrays hold: the stored vectors, their codes, norms, ids and lists, the trained arrays and the
 * tensor-core screening table; not the search workspace; the allocated capacity, so it includes
 * the headroom of a growing store, which dfx_reserve avoids) */
int dfx_get_param(dfx_index *idx, const char *name, double *value);
/* pre-size the shard for n_total vectors (optional; avoids regrowth while bulk loading) */
int dfx_reserve(dfx_index *idx, int64_t n_total);
/* fold pending adds into the inverted lists now (otherwise done by the next search) */
int dfx_finalize(dfx_index *idx, void *stream);

/* ---- THE HOT PATH: faiss_index.search(query_batch, top_k) index.py:257 ----
 * D float32[nq,k], I int64[nq,k], 1 <= k <= 4096 for every kind.  An IVF search with k > 1024
 * writes every probed vector's candidate and selects per query; it raises an error before launching
 * anything when the nprobe longest lists together exceed 2^24 vectors (128 MiB of candidates).
 * IVF_PQR: the IVF-PQ stage runs at k' = k * k_factor (at most 16384; k' > 1024 takes the candidate
 * rows), and the k' candidates are re-ranked and selected down to k; the same holds for the base
 * kind's stage of an index with refine_flat. */
int dfx_search(dfx_index *idx, int64_t nq, const float *x, int64_t k, float *D, int64_t *I);
int dfx_search_dev(dfx_index *idx, int64_t nq, const float *d_x, int64_t k, float *d_D,
                   int64_t *d_I, void *stream);

/* ---- range search: faiss_index.range_search(x, radius) of IndexFlat, IndexIVFFlat, IndexIVFPQ and
 * IndexIVFScalarQuantizer, made deterministic.
 * The vectors considered are the ones a dfx_search of the same shard scores: every row of FLAT,
 * the rows of the nprobe probed lists of IVF (same coarse quantizer, same nprobe clamping).  A
 * vector is returned when its distance D passes the radius strictly, as in faiss: D < radius for
 * L2, D > radius for inner product (a distance equal to the radius is excluded; NaN never
 * passes; +-inf radii are allowed, a NaN radius is refused).  The metric is the shard's SEARCH
 * metric: cfg.metric for FLAT, FLAT_SQ16, FLAT_PQ and IVF_FLAT, L2 for IVF_PQ, IVF_SQ16 and IVF_SQ8 (whose cfg.metric
 * is the coarse quantizer's).  Every returned (D, I) pair is bit for bit the pair dfx_search at a
 * large enough k reports for that id, and each query's results are sorted best first in the total
 * order of the search (ranking value ascending, then id ascending; inner product descending).
 * Served: FLAT, FLAT_SQ16, FLAT_PQ, IVF_FLAT, IVF_PQ (8- and 4-bit codes, every layout), IVF_SQ16, IVF_SQ8.  Refused
 * before anything is launched: IVF_PQ_FS (its distances are dequantized after the selection),
 * IVF_PQR and refine_flat (a radius over two stages of distances is not defined), an untrained IVF
 * or FLAT_PQ index.  Limits: an IVF query chunk's candidates obey the rule of k > 1024 (the nprobe longest
 * lists together at most 2^24 vectors), and one call returns at most 2^27 results; a call that
 * would return more raises once its counts are known, returns nothing, and leaves the shard
 * searchable (split the batch).
 * dfx_range_search: x host [nq, d], lims host int64[nq + 1]; the results of query i are entries
 * lims[i] .. lims[i + 1] - 1.  dfx_range_fetch then copies the lims[nq] entries into host D
 * float32 and I int64.  The results stay in index-owned workspace until the next search or range
 * search of the index, and can be fetched any number of times until then.
 * dfx_range_search_dev: device queries and device d_lims, *total = lims[nq] on the host; it reads
 * counts back, synchronising once per query chunk (FLAT, FLAT_SQ16, FLAT_PQ: per chunk and 32768-row
 * tile) and once at the end, so it cannot be captured in a CUDA graph.  dfx_range_fetch_dev maps the
 * results into device d_D / d_I on the stream. */
int dfx_range_search(dfx_index *idx, int64_t nq, const float *x, float radius, int64_t *lims);
int dfx_range_fetch(dfx_index *idx, float *D, int64_t *I);
int dfx_range_search_dev(dfx_index *idx, int64_t nq, const float *d_x, float radius, int64_t *d_lims,
                         int64_t *total, void *stream);
int dfx_range_fetch_dev(dfx_index *idx, float *d_D, int64_t *d_I, void *stream);

/* faiss_index.search_and_reconstruct: decode rows by id (index.py:255); id -1 -> NaN row
 * (refine_flat: the stored fp32 row, as faiss reconstructs from the refine index) */
int dfx_reconstruct(dfx_index *idx, int64_t n, const int64_t *ids, float *out);

/* device form, for winners that travelled through the all-gather + merge (client.py:287-289,
 * 299-307 carry per-shard embeddings to the client; here only the WINNERS are decoded, by the
 * shard that owns them).  shard_tag < 0: d_ids are shard-local ids, as dfx_reconstruct.
 * shard_tag >= 0: d_ids are exchange ids (dfx_encode_ids_dev); rows owned by another shard (or
 * empty, -1) are left untouched, so every rank decodes into a zeroed [n, d] buffer and the
 * buffers are summed. */
int dfx_reconstruct_dev(dfx_index *idx, int64_t n, const int64_t *d_ids, int64_t shard_tag,
                        float *d_out, void *stream);

/* ---- attributes the wrapper touches: .nprobe (index.py:356,495) .ntotal (index.py:184)
 *      .nlist / .quantizer.reconstruct_n(0, nlist) (index.py:350) ---- */
int dfx_set_nprobe(dfx_index *idx, int64_t nprobe);
int64_t dfx_get_nprobe(const dfx_index *idx);
int64_t dfx_ntotal(const dfx_index *idx);
/* changes whenever a call may have changed what a search launches (train / add / finalize /
 * import / set_param / set_nprobe); callers that replay captured CUDA graphs key them on it */
int64_t dfx_generation(const dfx_index *idx);
int64_t dfx_nlist(const dfx_index *idx);
int dfx_is_trained(const dfx_index *idx);
int dfx_get_centroids(dfx_index *idx, float *out /* [nlist, d] host */);

/* ---- cross-shard merge: faiss.float_maxheap_array_t as driven by ResultHeap /
 *      IndexClient._aggregate_results (client.py:29-54, 265-310).
 * D, I: [S][nq][k].  negate != 0 reproduces client.py:291-292 (search for -D when
 * metric == "dot"; the returned scores stay negated).  Keeps the k smallest, ascending;
 * an entry is admitted only if FLT_MAX > value (heapify() semantics); pads (FLT_MAX,-1).
 * outI[q][j] = I of the winner. */
int dfx_merge(int64_t S, int64_t nq, int64_t k, const float *D, const int64_t *I, int negate,
              float *outD, int64_t *outI);
int dfx_merge_dev(int64_t S, int64_t nq, int64_t k, const float *d_D, const int64_t *d_I,
                  int negate, float *d_outD, int64_t *d_outI, void *stream);

/* the same merge over what ONE all-gather of the ranks' result blocks delivers: rank r's block
 * starts at d_packed + r * rank_stride_bytes and holds D f32[S_loc][nq][k] at offset 0 and
 * I i64[S_loc][nq][k] at off_I_bytes (both multiples of 8).  Shard s = r * S_loc + j. */
int dfx_merge_packed_dev(int64_t R, int64_t S_loc, int64_t nq, int64_t k, const void *d_packed,
                         int64_t rank_stride_bytes, int64_t off_I_bytes, int negate,
                         float *d_outD, int64_t *d_outI, void *stream);

/* the cross-shard merge of range search results (IndexClient.range_search over the search plane).
 * Input: S shards' results of the same nq queries, concatenated shard-major: d_lims int64[S][nq + 1]
 * (each shard's own offsets, lims[s][0] = 0), d_D float32[total] and one int64 payload per entry d_P
 * [total] (ids or metadata codes; carried, never read), total = the sum of lims[s][nq].  Shard s's query q
 * holds entries base_s + lims[s][q] .. base_s + lims[s][q + 1] - 1, base_s = the totals of the shards
 * before s, and each such run must be sorted best first, as dfx_range_fetch returns it.
 * Output: d_out_lims int64[nq + 1], d_outD / d_outP [total] and d_order int64[total] (the input entry of
 * each output slot, to move embeddings or metadata the same way).  The order is that of a stable sort of
 * the concatenation by (query, score): per query best first -- maximize == 0: ascending (L2), != 0:
 * descending (inner product) --, equal scores by shard, then by the shard's own order.  Scores compare as
 * floats (-0 == +0) and are never negated; NaN must not occur (no NaN passes a radius).  Deterministic, no
 * atomics, graph-capturable (no read-back). */
int dfx_range_merge_dev(int64_t S, int64_t nq, const int64_t *d_lims, const float *d_D, const int64_t *d_P,
                        int64_t total, int maximize, int64_t *d_out_lims, float *d_outD, int64_t *d_outP,
                        int64_t *d_order, void *stream);

/* shard-local ids -> exchange ids: out = ids < 0 ? -1 : (shard_tag << 40) | ids, so that the
 * client can tell which (shard, local id) won after the merge (the reference's synthetic
 * positions, client.py:288).  d_col (optional): one int32 code per local id for ONE metadata
 * position (-2 = no metadata / tuple too short); entries whose code == drop_code or -2 are what
 * search_with_filter's post-filter drops (client.py:235-243) and get bit 62 set. */
int dfx_encode_ids_dev(int64_t n, const int64_t *d_ids, int64_t shard_tag, const int32_t *d_col,
                       int32_t drop_code, int64_t *d_out, void *stream);
/* search_with_filter's post-filter on device (client.py:229-250): per query, walk the k_in merged
 * slots in rank order, keep existing entries without the drop flag, stop at k_out; pads
 * (FLT_MAX, -1); d_count[q] = number kept. */
int dfx_filter_compact_dev(int64_t nq, int64_t k_in, int64_t k_out, const float *d_D,
                           const int64_t *d_I, float *d_outD, int64_t *d_outI, int32_t *d_count,
                           void *stream);

/* map shard-local ids to caller ids on device: out[i] = ids[i] < 0 ? -1 : table[ids[i]]
 * (the device form of Index.search's id -> metadata loop, index.py:260-268, for the
 * integer-metadata convention of scripts/load_data.py:120-124). */
int dfx_map_ids_dev(int64_t n, const int64_t *d_ids, const int64_t *d_table, int64_t *d_out,
                    void *stream);

/* ---- state exchange (tests, persistence; not on the timed path) ----
 * named arrays, host memory, list-sorted storage order:
 *   "centroids" f32[nlist,d]   "codebooks" f32[M,ksub,dsub]   "list_off" i64[nlist+1]
 *   "ids" i64[ntotal]   "codes" u8[ntotal,M]   "tvals" f32[ntotal]
 *   (IVF_PQ: "codes" holds one code per byte whatever pq_nbits is, and "codebooks" has ksub =
 *   1 << pq_nbits; 4-bit codes are packed and unpacked on the way, and an imported code >= 16 is
 *   refused)
 *   (IVF_PQ_FS: "centroids", "codebooks" f32[M,16,dsub], "list_off", "ids" and "codes" u8[ntotal,M],
 *   one 4-bit code per byte as for IVF_PQ; no "tvals", since the codes are not residuals)
 *   "vecs" f32[ntotal,d] (IVF_FLAT)   "codes16" u16[ntotal,d]   "xb" f32[ntotal,d] (FLAT)
 *   (FLAT_SQ16: "codes16" alone, the fp16 rows in id order; like "xb" its import sets ntotal)
 *   (FLAT_PQ: "codebooks" f32[M,256,dsub], then "codes" u8[ntotal,M] in id order, whose import sets
 *   ntotal)
 *   "sq_trained" f32[2,d] (IVF_SQ8: vmin, then vdiff -- faiss's ScalarQuantizer::trained)
 *   "codes8" u8[ntotal,d] (IVF_SQ8)
 *   (IVF_PQR: the IVF_PQ arrays with 8-bit codes, plus "refine_codebooks" f32[M2,256,d/M2] and
 *   "refine_codes" u8[ntotal,M2] in ID order, not list order; its "ids" must be a permutation of
 *   0 .. ntotal-1, and "tvals" is recomputed on import)
 *   (refine_flat: the base kind's arrays, plus "refine_vecs" f32[ntotal,d] in ID order; "ids" must
 *   be a permutation of 0 .. ntotal-1, and "refine_vecs" follows the payload on import)
 * dfx_get_array with out == NULL only reports the size.  Import order: centroids,
 * codebooks (IVF_PQ, IVF_PQ_FS, IVF_PQR) or sq_trained (IVF_SQ8), refine_codebooks (IVF_PQR), then
 * list_off, ids and the payload, refine_codes (IVF_PQR), then dfx_import_done(). */
int dfx_get_array(dfx_index *idx, const char *name, void *out, int64_t max_bytes,
                  int64_t *nbytes);
int dfx_set_array(dfx_index *idx, const char *name, const void *in, int64_t nbytes);
int dfx_import_done(dfx_index *idx);

/* statistics of the most recent search or range search (device work, synchronises):
 * ndis = sum over (query, probed list) of the list length -- faiss's `ndis` (IVF_PQR: of the
 * IVF-PQ stage, refine_flat: of the base kind's stage; the re-ranked candidates are not counted). */
int dfx_last_stats(dfx_index *idx, int64_t *ndis, int64_t *nq, int64_t *nprobe);
/* per-kernel timing of the dominant kernel (the inverted-list scan): when enabled, every scan
 * launch is bracketed by CUDA events on the launching stream; dfx_profile_read synchronises
 * those events and returns the summed device time and the number of launches. */
int dfx_profile_enable(dfx_index *idx, int on);
int dfx_profile_read(dfx_index *idx, double *scan_ms, int64_t *scan_launches, int reset);
/* number of kernel launches issued by this library since process start */
int64_t dfx_launch_count(void);

/* ---- synthetic data on device (bench harness; SURVEY.md 8d generator, see DESIGN.md) ----
 * x_i = mu_{c(i)} + A (sigma * z_{g(i)} + delta * w_i) + eps * n_i
 *   C cluster centres mu_c ~ N(0, I_d);  c(i) = i mod C
 *   G groups ("near-duplicate" micro-clusters), g(i) = i mod G (G multiple of C; G = 0: one
 *   group per row); latent z_g ~ N(0, I_r) clipped to |z| <= 4;  A: d x r, orthonormal columns
 *   w_i ~ N(0, I_r), n_i ~ N(0, I_d) per row.
 * Counter-based: any row is regenerable anywhere from (seed, row).  rows: optional explicit row
 * ids (else row0 .. row0+n-1).  noise_stream != 0 adds sigma_q * N(0, I_d) (queries). */
typedef struct dfx_synth {
    uint64_t seed;
    int32_t d;
    int32_t r;        /* intrinsic dimension of the cluster-level structure */
    int64_t nclusters;
    int64_t ngroups;
    float sigma;
    float eps;
    float sigma_q;
    float delta;
} dfx_synth;
int dfx_synth_init(const dfx_synth *p, float **d_A_out /* device [d,r], caller frees with dfx_free */,
                   void *stream);
int dfx_synth_rows_dev(const dfx_synth *p, const float *d_A, int64_t row0, const int64_t *d_rows,
                       int64_t n, uint64_t noise_stream, float *d_out, void *stream);
int dfx_free(void *d_ptr);

const char *dfx_last_error(void);
const char *dfx_version(void);
/* byte offset, inside a 1 KB block of 32 IVF-PQ vectors, of subquantizer m of vector v for block
 * layout 1 or 2 (host function; lets the layout be checked without a GPU) */
int dfx_debug_il_byte(int layout, int v, int m);
/* the coarse quantizer's tensor-core screening summary of nq device queries d_x [nq, d] against
 * the centroids of a trained IVF index (d a multiple of 64), at npl = 1 (FAST) or 2 (PRECISE)
 * fp16 planes: per query and group of 32 centroids, the smallest ranking value with the winning
 * column (0..31) in its 5 low bits (d_gmin), the runner-up (d_gmin2) and that column (d_gargc);
 * device arrays of [nq][ceil(nlist / 128) * 4].  Synchronises. */
int dfx_debug_tc_screen(dfx_index *idx, int64_t nq, const float *d_x, int npl, float *d_gmin, float *d_gmin2,
                        uint8_t *d_gargc);

#ifdef __cplusplus
}
#endif
#endif /* DFX_H */
