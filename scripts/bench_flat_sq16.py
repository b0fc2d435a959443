#!/usr/bin/env python
"""fp32 flat against "SQfp16" (IndexScalarQuantizer QT_fp16) on the same rows, one H100, inner product.

Rows: the bench generator (kind_bench.Dataset "bench": near-duplicate groups of 10) at d = 768, added
on the device in steps of 250 000.  Two shards of N = 5 M rows: FLAT (fp32 rows + the fp16 hi/lo
screening planes) and FLAT_SQ16 (the fp16 rows only), then one FLAT_SQ16 shard of N = 21 M rows (the
DPR Wikipedia passage count), which an fp32 flat shard cannot hold on one 80 GB card.
Per shard and case (nq in {1, 64, 1024, 4096}, k in {10, 100}), with device-resident queries through
search_dev:
  batch_ms    one call, device-synchronised (CUDA events, kind_bench.timed: warm-up, then the mean of
              `iters` calls), the median over `rounds` rounds
  qps         nq / batch_ms
and per shard index_bytes / N (dfx_get_param "index_bytes", after the first search built the screening
table).  recall_at_k: the fraction of the fp32 flat shard's k ids per query that the SQfp16 shard of the
same rows returns.  The card name and its power limit are recorded with the numbers."""
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

NQS, KS = (1, 64, 1024, 4096), (10, 100)


def log(msg):
    print(msg, file=sys.stderr, flush=True)


def time_cases(g, xq, rounds, iters):
    out = {}
    for nq in NQS:
        q = xq[:nq].contiguous()
        for k in KS:
            D = torch.empty((nq, k), dtype=torch.float32, device="cuda")
            I = torch.empty((nq, k), dtype=torch.int64, device="cuda")
            ms = float(np.median([kb.timed(lambda: g.search_dev(q, k, D, I), iters=iters, warm=2)
                                  for _ in range(rounds)]))
            out[f"nq{nq}_k{k}"] = {"batch_ms": ms, "qps": nq / ms * 1e3}
            log(f"  nq={nq} k={k}: {ms:.3f} ms")
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=5_000_000)
    ap.add_argument("--n-large", type=int, default=21_000_000)
    ap.add_argument("--d", type=int, default=768)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--iters", type=int, default=5)
    a = ap.parse_args()
    d, n = a.d, a.n
    out = {"card": kb.card(), "setup": {"d": d, "n": n, "n_large": a.n_large, "metric": "IP", "nq": NQS, "k": KS,
                                        "rounds": rounds_iters(a), "dataset": "bench (near-duplicate groups of 10)"}}
    ds = kb.Dataset(d, n, max(NQS), step=250_000)
    xq = ds.xq.contiguous()
    shards = {}
    for name, kind in (("flat", engine.KIND_FLAT), ("sq16", engine.KIND_FLAT_SQ16)):
        g = engine.GpuIndex(kind, d, engine.METRIC_INNER_PRODUCT)
        g.reserve(n)
        for r0 in range(0, n, ds.step):
            g.add_dev(ds.synth.rows(r0, min(ds.step, n - r0)))
        torch.cuda.synchronize()
        g.search_dev(xq[:1], 10)
        torch.cuda.synchronize()
        shards[name] = g
        out[name] = {"index_bytes_per_vector": g.get_param("index_bytes") / n}
        log(f"{name}: {n} rows added, {out[name]['index_bytes_per_vector']:.1f} B/vector")
    recall = {}
    for k in KS:
        _, If = shards["flat"].search_dev(xq, k)
        _, Is = shards["sq16"].search_dev(xq, k)
        If, Is = If.cpu().numpy(), Is.cpu().numpy()
        recall[f"k{k}"] = float(np.mean([len(np.intersect1d(a, b)) / k for a, b in zip(If, Is)]))
    out["recall_at_k_sq16_vs_flat"] = recall
    log(f"recall {recall}")
    for name, g in shards.items():
        log(name)
        out[name]["cases"] = time_cases(g, xq, a.rounds, a.iters)
    del shards
    torch.cuda.empty_cache()

    if a.n_large > 0:
        big = kb.Dataset(d, a.n_large, max(NQS), step=250_000)
        g = engine.GpuIndex(engine.KIND_FLAT_SQ16, d, engine.METRIC_INNER_PRODUCT)
        g.reserve(a.n_large)
        for r0 in range(0, a.n_large, big.step):
            g.add_dev(big.synth.rows(r0, min(big.step, a.n_large - r0)))
        torch.cuda.synchronize()
        g.search_dev(big.xq[:1].contiguous(), 10)
        torch.cuda.synchronize()
        out["sq16_large"] = {"n": a.n_large, "index_bytes_per_vector": g.get_param("index_bytes") / a.n_large,
                             "cases": time_cases(g, big.xq.contiguous(), a.rounds, a.iters)}
    print(json.dumps(out, indent=1))


def rounds_iters(a):
    return {"rounds": a.rounds, "iters": a.iters}


if __name__ == "__main__":
    main()
