// dfx_scan_il2.cu -- launcher of the IVF-PQ (M == 32) table build + inverted-list scan, K3 + K4.
// Kernel: dfx_scan_il2_dev.cuh.
#include "dfx_scan_il2_dev.cuh"
#include <cstdlib>

// dynamic shared memory of one CTA: the query's table + one queue (REG) or WarpTopK buffer per warp
static size_t il2_smem(bool reg, int threads, int cap) {
    return (size_t)IL2_LUT_BYTES + (size_t)(threads / 32) * (reg ? IL2_QCAP : cap) * 8;
}

// blocks the L2 prefetch cursor runs ahead of the register loads (0 = off; DFX_IL2_PREFETCH)
static int il2_pf_ahead(const dfx_index* idx) {
    static const int pf_default = [] {
        const char* e = getenv("DFX_IL2_PREFETCH");
        const int v = e ? atoi(e) : 4;
        return v < 0 ? 0 : (v > 32 ? 32 : v);
    }();
    return idx->il2_prefetch >= 0 ? idx->il2_prefetch : pf_default;
}

template <bool REG, int THREADS, int MINB>
static void launch_il2_t(dfx_index* idx, const float* xq, int64_t qc, const int32_t* keys, int nprobe, int G,
                       int ngroups, int k, int cap, uint64_t* part, float* outD, int64_t* outI, cudaStream_t st) {
    const size_t smem = il2_smem(REG, THREADS, cap);
    auto kern = scan_pq_il2_kernel<REG, THREADS, MINB>;
    DFX_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    DFX_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributePreferredSharedMemoryCarveout, 100));
    const int pf_ahead = il2_pf_ahead(idx);
    DFX_LAUNCH(kern, (unsigned)(qc * ngroups), THREADS, smem, st, xq, idx->codebooksT.as<float>(),
               idx->centroids.as<float>(), idx->cfg.d, idx->dsub, keys, nprobe, G, ngroups, idx->blk_off.as<int64_t>(),
               idx->il_codes.as<uint4>(), idx->il_tvals.as<float>(), idx->il_ids.as<int32_t>(), k, cap, part, outD, outI,
               pf_ahead, (const int64_t*)nullptr);
}

// CTA shape: 256 threads x 3 CTAs per SM (default) or, DFX_IL2_THREADS=512, 512 threads x 2 CTAs
// (16 warps share one query's table: 32 instead of 24 warps per SM, half the table builds per SM).
// 512 threads at k > 512 would need 16 buffers of cap = 2048 composites (320 KB): more than one CTA
// may opt in to, so those searches take the 256-thread shape.
template <bool REG>
static void launch_il2(dfx_index* idx, const float* xq, int64_t qc, const int32_t* keys, int nprobe, int G,
                       int ngroups, int k, int cap, uint64_t* part, float* outD, int64_t* outI, cudaStream_t st) {
    static const int threads_default = [] {
        const char* e = getenv("DFX_IL2_THREADS");
        return e ? atoi(e) : IL2_THREADS;
    }();
    const int threads = idx->il2_threads ? idx->il2_threads : threads_default;
    if (threads == 512 && il2_smem(REG, 512, cap) <= (size_t)dfx_smem_optin()) launch_il2_t<REG, 512, 2>(idx, xq, qc, keys, nprobe, G, ngroups, k, cap, part, outD, outI, st);
    else launch_il2_t<REG, 256, 3>(idx, xq, qc, keys, nprobe, G, ngroups, k, cap, part, outD, outI, st);
}

// outD / outI: when ngroups == 1 and k <= 32 the kernel writes the final rows there and the
// function returns true (the caller skips the per-query reduction of `part`).
static void il2_prepare(dfx_index* idx, int G, cudaStream_t st) {
    DFX_REQUIRE(G <= IL2_MAXG, "scan_pq_il2: more than 16 probes per CTA");
    DFX_REQUIRE(idx->M == 32 && idx->ksub == 256 && idx->cfg.d == 32 * idx->dsub, "scan_pq_il2: M == 32 x 8 bit only");
    if (!idx->cbT_valid) {  // transposed codebook PT[j][m][dsub], once per trained / imported codebook
        const int tot = idx->M * idx->ksub * idx->dsub;
        idx->codebooksT.reserve((size_t)tot * 4);
        DFX_LAUNCH(cb_transpose_kernel, (unsigned)((tot + 255) / 256), 256, 0, st, idx->codebooks.as<float>(), idx->M,
                   idx->ksub, idx->dsub, idx->codebooksT.as<float>());
        idx->cbT_valid = true;
    }
}

bool dfx_launch_scan_pq_il2(dfx_index* idx, const float* xq, int64_t qc, const int32_t* keys, int nprobe, int G,
                            int ngroups, int k, int cap, uint64_t* part, float* outD, int64_t* outI,
                            cudaStream_t st) {
    il2_prepare(idx, G, st);
    const bool reg = k <= 32;
    const bool direct = reg && ngroups == 1 && outD != nullptr;
    if (reg) launch_il2<true>(idx, xq, qc, keys, nprobe, G, ngroups, k, cap, part, direct ? outD : nullptr,
                              direct ? outI : nullptr, st);
    else launch_il2<false>(idx, xq, qc, keys, nprobe, G, ngroups, k, cap, part, nullptr, nullptr, st);
    return direct;
}

// k > 1024: every vector's composite to its slot of the candidate rows (cand, offsets coff).  Always
// the 256-thread shape; its shared memory is the table and the probes' slot bases.
void dfx_launch_scan_pq_il2_mat(dfx_index* idx, const float* xq, int64_t qc, const int32_t* keys, int nprobe, int G,
                                int ngroups, uint64_t* cand, const int64_t* coff, cudaStream_t st) {
    il2_prepare(idx, G, st);
    const size_t smem = (size_t)IL2_LUT_BYTES + (size_t)2 * IL2_MAXG * 8;
    auto kern = scan_pq_il2_kernel<false, 256, 3, true>;
    DFX_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    DFX_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributePreferredSharedMemoryCarveout, 100));
    const int pf_ahead = il2_pf_ahead(idx);
    DFX_LAUNCH(kern, (unsigned)(qc * ngroups), 256, smem, st, xq, idx->codebooksT.as<float>(), idx->centroids.as<float>(),
               idx->cfg.d, idx->dsub, keys, nprobe, G, ngroups, idx->blk_off.as<int64_t>(), idx->il_codes.as<uint4>(),
               idx->il_tvals.as<float>(), idx->il_ids.as<int32_t>(), 0, 0, cand, (float*)nullptr, (int64_t*)nullptr,
               pf_ahead, coff);
}
