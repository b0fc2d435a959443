#!/usr/bin/env python
"""Range search against k-NN search on one 8-bit IVF-PQ shard (one H100).

Shard: the bench generator (kind_bench.Dataset "bench": rows in near-duplicate groups of 10) at
d = 128, 2M vectors, nlist 2048, M = 32 (the interleaved block scan), nprobe 32, 1 000 queries.  The
radii come from a k-NN run: the median over the queries of the 10th and of the 100th L2 distance,
aiming at about 10 and 100 results per query (the means are reported; the groups of 10 put a gap in
the distances after the 10th neighbour, so the second radius returns more).  Per case, on the same
host queries through the host entry points (query upload and result download included):
  batch_ms          one call over the 1 000 queries (CUDA events around calls that end in a
                    synchronise, median over rounds; warm-up as kind_bench.timed)
  results_per_query mean results per query (range) or k (search)
  ndis              the probed vectors the call scored (dfx_last_stats)
Before any time is taken, each radius's results must equal the k-NN search at k = the largest count of
any query + 1 (at most 4096), cut at the radius, for every query whose count is below that k.
The card name and its power limit are recorded with the numbers."""
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import kind_bench as kb  # noqa: E402
from distributed_faiss_b200 import engine  # noqa: E402


def check_against_cut_search(g, xq, radius):
    """range results == search(k) cut at radius for every query with fewer than k results"""
    lims, D, I = g.range_search(xq, radius)
    cnt = np.diff(lims)
    k = int(min(4096, cnt.max() + 1))
    Ds, Is = g.search(xq, k)
    ok = cnt < k
    keep = (Is >= 0) & (Ds < np.float32(radius))
    same = all(np.array_equal(I[lims[q]:lims[q + 1]], Is[q][keep[q]]) and
               np.array_equal(D[lims[q]:lims[q + 1]].view(np.int32), Ds[q][keep[q]].view(np.int32))
               for q in np.nonzero(ok)[0])
    return bool(same), int(ok.sum())


def main():
    d, n, nlist, M, nprobe, nq = 128, 2_000_000, 2048, 32, 32, 1000
    rounds = 3
    out = {"card": kb.card(), "setup": {"d": d, "n": n, "nlist": nlist, "M": M, "nprobe": nprobe, "nq": nq,
                                        "rounds": rounds, "dataset": "bench (near-duplicate groups of 10)"}}
    ds = kb.Dataset(d, n, nq, step=500_000)
    g = ds.fill(engine.GpuIndex(engine.KIND_IVF_PQ, d, engine.METRIC_L2, nlist=nlist, pq_m=M), nlist, nprobe)
    xq = ds.xq.cpu().numpy()
    Dk, _ = g.search(xq, 100)
    radii = {"range_r10": float(np.median(Dk[:, 9])), "range_r100": float(np.median(Dk[:, 99]))}

    calls, res = {}, {}
    for name, r in radii.items():
        same, checked = check_against_cut_search(g, xq, r)
        if not same:
            raise SystemExit(f"{name}: range search differs from the cut k-NN search")
        lims, _, _ = g.range_search(xq, r)
        res[name] = {"radius": r, "results_per_query": float(lims[-1]) / nq, "max_results": int(np.diff(lims).max()),
                     "checked_queries": checked, "ndis": g.last_stats()["ndis"]}
        calls[name] = (lambda r=r: g.range_search(xq, r))
    for k in (10, 100):
        g.search(xq, k)
        res[f"search_k{k}"] = {"results_per_query": k, "ndis": g.last_stats()["ndis"]}
        calls[f"search_k{k}"] = (lambda k=k: g.search(xq, k))
    for name in calls:
        res[name]["batch_ms_rounds"] = []
    for _ in range(rounds):
        for name, fn in calls.items():
            res[name]["batch_ms_rounds"].append(kb.timed(fn))
    for r in res.values():
        r["batch_ms"] = float(np.median(r["batch_ms_rounds"]))
    out.update(res)
    print(json.dumps(out, indent=1))


if __name__ == "__main__":
    main()
