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
import kind_bench as kb  # noqa: E402
from distributed_faiss_b200 import engine  # noqa: E402
from oracle import oracle as O  # noqa: E402


def main():
    d, n, nlist, nprobe, nq, k = 768, 2_000_000, 2048, 32, 1000, 10
    out = {"card": kb.card(), "setup": {"d": d, "n": n, "nlist": nlist, "nprobe": nprobe, "nq": nq, "k": k}}
    ds = kb.Dataset(d, n, nq, step=500_000, seed=99, r=32)
    ds.exact(k)
    xs = ds.sample()

    cent0 = None
    for M in (64, 96, 128):
        g = ds.fill(engine.GpuIndex(engine.KIND_IVF_PQ, d, engine.METRIC_L2, nlist=nlist, pq_m=M), nlist, nprobe)
        cent = g.get_centroids()
        if cent0 is None:
            cent0 = cent
        batch_ms, scan_ms, _, ndis = kb.measure(g, ds.xq, k, reps=10)
        recall = ds.recall(g, k)
        o = O.make_index("ivf_pq", d, metric=O.METRIC_L2, nlist=nlist, M=M)
        out[f"M{M}"] = {
            "batch_ms": batch_ms, "qps": nq / batch_ms * 1e3, "scan_kernel_ms": scan_ms, "ndis": ndis,
            "lookups_per_s": ndis * M / (scan_ms * 1e-3), "code_GBps": ndis * M / (scan_ms * 1e-3) / 1e9,
            "recall_at_10": recall, "same_centroids_as_M64": bool(np.array_equal(cent, cent0)),
            "bit_exact_vs_oracle_32q": kb.same_arrays(g.search(xs, k), kb.mirror(o, g, nprobe).search(xs, k)),
        }
        print(json.dumps({f"M{M}": out[f"M{M}"]}), flush=True)
        del g, o
        torch.cuda.empty_cache()
    print(json.dumps(out, indent=1))


if __name__ == "__main__":
    main()
