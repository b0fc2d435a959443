#!/usr/bin/env python
"""IVF-PQ at M = 64, 96 and 128 on one H100: the row-major scan at M = 64 (scan_pq_kernel<64>) and
the wide-code scan above it (scan_pq_wide_kernel, table built in shared memory).

Shard: synthetic d = 768 (the bench generator), 2M vectors, nlist 2048, 1 000 queries, nprobe 32,
k = 10.  The coarse k-means runs with the same seed on the same rows for every M, so the shards
hold the same centroids and lists (checked and reported); only the codes differ.  Per M:
  batch_ms         one search of the 1 000 device-resident queries (CUDA events, 3 warm-ups)
  scan_kernel_ms   the list-scan launch alone (dfx_profile_*: the table + |q - c|^2 preparation and
                   the scan, bracketed by CUDA events)
  lookups_per_s    ndis x M table lookups over scan_kernel_ms
  code_GBps        ndis x M code bytes over scan_kernel_ms
  recall_at_10     against the exact top-10 of the GPU flat (L2) index over the same 2M vectors
  bit_exact_vs_oracle_32q  a query sample against the oracle holding the same shard state
The card name and its power limit are recorded with the numbers."""
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))
from bench_other_configs import card, timed  # noqa: E402
from distributed_faiss_b200 import engine  # noqa: E402
from oracle import oracle as O  # noqa: E402


def main():
    d, n, nlist, nprobe, nq, k = 768, 2_000_000, 2048, 32, 1000, 10
    step = 500_000
    out = {"card": card(), "setup": {"d": d, "n": n, "nlist": nlist, "nprobe": nprobe, "nq": nq, "k": k}}
    synth = engine.Synth(99, d, 32, 1, 1.0, 0.02, ngroups=n // 10, eps=0.01, delta=0.1)
    rows = torch.randint(0, n, (nq,), dtype=torch.int64, generator=torch.Generator().manual_seed(1)).cuda()
    xq_t = synth.rows(0, nq, rows_t=rows, noise_stream=7)

    flat = engine.GpuIndex(engine.KIND_FLAT, d, engine.METRIC_L2)
    flat.reserve(n)
    for r0 in range(0, n, step):
        flat.add_dev(synth.rows(r0, min(step, n - r0)))
    exact = flat.search_dev(xq_t, k)[1].cpu().numpy()
    del flat
    torch.cuda.empty_cache()

    cent0 = None
    for M in (64, 96, 128):
        g = engine.GpuIndex(engine.KIND_IVF_PQ, d, engine.METRIC_L2, nlist=nlist, pq_m=M)
        g.set_param("kmeans_niter", 10)
        g.set_param("max_points_per_centroid", 64)
        g.train_dev(synth.rows(0, 64 * nlist))
        for r0 in range(0, n, step):
            g.add_dev(synth.rows(r0, min(step, n - r0)))
        g.finalize()
        g.nprobe = nprobe
        cent = g.get_centroids()
        if cent0 is None:
            cent0 = cent
        batch_ms = timed(lambda: g.search_dev(xq_t, k))
        g.profile(True)
        reps = 10
        for _ in range(reps):
            g.search_dev(xq_t, k)
        torch.cuda.synchronize()
        scan_ms, launches = g.profile_read()
        g.profile(False)
        scan_ms /= reps
        ndis = g.last_stats()["ndis"]
        I = g.search_dev(xq_t, k)[1].cpu().numpy()
        recall = float(np.mean([len(set(a) & set(b)) / k for a, b in zip(I, exact)]))
        xs = xq_t[:32].cpu().numpy()
        Dg, Ig = g.search(xs, k)
        o = O.make_index("ivf_pq", d, metric=O.METRIC_L2, nlist=nlist, M=M)
        o.set_state(g.get_state())
        o.nprobe = nprobe
        Do, Io = o.search(xs, k)
        out[f"M{M}"] = {
            "batch_ms": batch_ms, "qps": nq / batch_ms * 1e3, "scan_kernel_ms": scan_ms, "ndis": ndis,
            "lookups_per_s": ndis * M / (scan_ms * 1e-3), "code_GBps": ndis * M / (scan_ms * 1e-3) / 1e9,
            "recall_at_10": recall, "same_centroids_as_M64": bool(np.array_equal(cent, cent0)),
            "bit_exact_vs_oracle_32q": bool(np.array_equal(Dg, Do) and np.array_equal(Ig, Io)),
        }
        print(json.dumps({f"M{M}": out[f"M{M}"]}), flush=True)
        del g, o
        torch.cuda.empty_cache()
    print(json.dumps(out, indent=1))


if __name__ == "__main__":
    main()
