#!/usr/bin/env python
"""Product-quantized flat shards ("PQ{M}", faiss IndexPQ(d, M, 8, metric)) on one H100.

Rows: the bench generator (kind_bench.Dataset "bench": near-duplicate groups of 10), added on the device
in steps of 250 000, N = 10 M per shard.  Configurations: d = 768 under inner product (the default metric
of IndexCfg) with M in {32, 64, 96}, d = 768 under L2 with M = 64 (the same rows under the other metric), and
d = 128 under L2 with M = 32.  Each shard is trained on its first
65 536 rows (kmeans_niter iterations per sub-quantizer).
Per shard and case (nq in {1, 64, 1024}, k in {10, 100, 1024, 1025}), with device-resident queries through
search_dev:
  batch_ms          one call, device-synchronised (CUDA events, kind_bench.timed: warm-up, then the mean of
                    `iters` calls), the median over `rounds` rounds.  The search picks its path by (nq, k):
                    the fused per-tile top-k for k <= 100 or nq * k <= 16384 (the cases with k <= 100,
                    and k = 1024 at nq = 1), the values tiles otherwise (k = 1024 at nq >= 64, and k = 1025)
  qps               nq / batch_ms
  code_share_hbm    nq = 1 only: N * M code bytes per batch_ms, as a share of the H100 SXM data-sheet
                    bandwidth, 3.35 TB/s
and per shard index_bytes / N (dfx_get_param "index_bytes") and recall@k of the first 64 queries against
an exact fp32 flat search of the same rows (a FLAT shard on the FFMA path, built and freed per
configuration).  The card name and its power limit are recorded with the numbers."""
import argparse
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import kind_bench as kb  # noqa: E402
from distributed_faiss_b200 import engine  # noqa: E402

NQS, KS = (1, 64, 1024), (10, 100, 1024, 1025)
CONFIGS = [(768, engine.METRIC_INNER_PRODUCT, (32, 64, 96)), (768, engine.METRIC_L2, (64,)), (128, engine.METRIC_L2, (32,))]
HBM_BYTES_PER_S = 3.35e12
RECALL_NQ = 64


def log(msg):
    print(msg, file=sys.stderr, flush=True)


def exact_ids(ds, metric, k):
    """the exact top-k ids of the first RECALL_NQ queries (fp32 flat on the FFMA path: no screening planes)"""
    flat = engine.GpuIndex(engine.KIND_FLAT, ds.d, metric)
    flat.set_param("flat_tensor_cores", 0)
    flat.reserve(ds.n)
    ds.add(flat)
    ids = flat.search_dev(ds.xq[:RECALL_NQ].contiguous(), k)[1].cpu().numpy()
    del flat
    torch.cuda.empty_cache()
    return ids


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=10_000_000)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--niter", type=int, default=10, help="k-means iterations per sub-quantizer")
    a = ap.parse_args()
    n = a.n
    out = {"card": kb.card(), "setup": {"n": n, "nq": NQS, "k": KS, "rounds": a.rounds, "iters": a.iters,
                                        "kmeans_niter": a.niter, "train_rows": 65536,
                                        "dataset": "bench (near-duplicate groups of 10)"}, "shards": []}
    for d, metric, Ms in CONFIGS:
        ds = kb.Dataset(d, n, max(NQS), step=250_000)
        exact = exact_ids(ds, metric, max(KS))
        for M in Ms:
            g = engine.GpuIndex(engine.KIND_FLAT_PQ, d, metric, pq_m=M)
            g.set_param("kmeans_niter", a.niter)
            g.train_dev(ds.synth.rows(0, 65536))
            g.reserve(n)
            ds.add(g)
            torch.cuda.synchronize()
            res = {"d": d, "metric": "IP" if metric == engine.METRIC_INNER_PRODUCT else "L2", "M": M,
                   "index_bytes_per_vector": g.get_param("index_bytes") / n, "recall_at_k": {}, "cases": {}}
            q64 = ds.xq[:RECALL_NQ].contiguous()
            for k in KS:
                I = g.search_dev(q64, k)[1].cpu().numpy()
                res["recall_at_k"][f"k{k}"] = float(np.mean([len(np.intersect1d(x, y)) / k
                                                             for x, y in zip(I, exact[:, :k])]))
            log(f"d={d} M={M}: {res['index_bytes_per_vector']:.2f} B/vector, recall {res['recall_at_k']}")
            for nq in NQS:
                q = ds.xq[:nq].contiguous()
                for k in KS:
                    D = torch.empty((nq, k), dtype=torch.float32, device="cuda")
                    I = torch.empty((nq, k), dtype=torch.int64, device="cuda")
                    ms = float(np.median([kb.timed(lambda: g.search_dev(q, k, D, I), iters=a.iters, warm=2)
                                          for _ in range(a.rounds)]))
                    case = {"batch_ms": ms, "qps": nq / ms * 1e3}
                    if nq == 1:
                        case["code_share_hbm"] = n * M / (ms * 1e-3) / HBM_BYTES_PER_S
                    res["cases"][f"nq{nq}_k{k}"] = case
                    log(f"  nq={nq} k={k}: {ms:.3f} ms")
            out["shards"].append(res)
            del g
            torch.cuda.empty_cache()
        del ds
        torch.cuda.empty_cache()
    print(json.dumps(out, indent=1))


if __name__ == "__main__":
    main()
