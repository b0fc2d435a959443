#!/usr/bin/env python
"""IVF-PQR ("IVF{n},PQ{M}+{M2}": the IVF-PQ search for k' = 4k candidates, re-ranked on the
reconstruction c + PQ1 + PQ2 by pqr_refine_kernel) against plain 8-bit IVF-PQ on one H100.

Shards: d = 128, nlist 4096, nprobe 32, 1 000 device-resident queries, k = 10, on two datasets of
PQR_BENCH_N (default 10M) vectors each:
  bench      the bench generator (bench.py's defaults: near-duplicate groups, low intrinsic dimension)
  clustered  the same generator as plain clustered data: 10 000 Gaussian clusters in 16 dimensions,
             no near-duplicate groups, per-row noise in all 128
The coarse k-means runs with the same seed on the same rows for every case, so every shard of one
dataset holds the same centroids and lists (checked and reported).  Cases:
  PQ16      scan_pq_kernel<16>                 16 B code + 4 B t-value + 4 B id per vector
  PQ16+16   the same scan at k' = 40, then the re-ranking of 40 candidates per query (16 B more per
            vector, stored by id and read only for the candidates)
  PQ32      the interleaved M = 32 scan        32 B code + 4 B t-value + 4 B id
The shards of a dataset stay resident and are timed in alternating rounds.  Per case:
  batch_ms         one search of the 1 000 queries (CUDA events, median over rounds)
  scan_kernel_ms   the first-stage list scan (dfx_profile_*: bracketed by CUDA events), median and
                   [min, max] over rounds
  refine_ms        PQ16+16 only: the re-ranking kernel + its final selection (dfx_get_param
                   "refine_ms"), median and [min, max] over rounds
  recall_at_10     against the exact top-10 of the GPU flat (L2) index over the same vectors
  bit_exact_vs_oracle_32q  a query sample against the oracle holding the same shard state
The card name and its power limit are read in the same run and recorded with the numbers."""
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
from tests.oracle_pqr import OracleIVFPQR  # noqa: E402

CASES = (("PQ16", 16, 0), ("PQ16+16", 16, 16), ("PQ32", 32, 0))
DATASETS = {
    "bench": dict(r=16, nclusters=1, sigma=1.0, sigma_q=0.02, eps=0.01, delta=0.1, groups_per=10),
    "clustered": dict(r=16, nclusters=10_000, sigma=1.0, sigma_q=0.05, eps=0.3, delta=0.0, groups_per=0),
}


def run_dataset(name, p, d, n, nlist, nprobe, nq, k, rounds, reps, step=1_000_000):
    ngroups = max(1, n // p["groups_per"]) if p["groups_per"] else 0
    if ngroups:
        ngroups = max(p["nclusters"], ngroups // p["nclusters"] * p["nclusters"])
    synth = engine.Synth(1234, d, p["r"], p["nclusters"], p["sigma"], p["sigma_q"], ngroups=ngroups, eps=p["eps"],
                         delta=p["delta"])
    rows = torch.randint(0, n, (nq,), dtype=torch.int64, generator=torch.Generator().manual_seed(1)).cuda()
    xq_t = synth.rows(0, nq, rows_t=rows, noise_stream=7)

    flat = engine.GpuIndex(engine.KIND_FLAT, d, engine.METRIC_L2)
    flat.reserve(n)
    for r0 in range(0, n, step):
        flat.add_dev(synth.rows(r0, min(step, n - r0)))
    exact = flat.search_dev(xq_t, k)[1].cpu().numpy()
    del flat
    torch.cuda.empty_cache()

    shards, res = {}, {}
    cent0 = off0 = None
    for case, M, M2 in CASES:
        kind = engine.KIND_IVF_PQR if M2 else engine.KIND_IVF_PQ
        g = engine.GpuIndex(kind, d, engine.METRIC_L2, nlist=nlist, pq_m=M, pq_nbits=8, refine_m=M2)
        g.set_param("kmeans_niter", 10)
        g.set_param("max_points_per_centroid", 64)
        g.train_dev(synth.rows(0, 64 * nlist))
        for r0 in range(0, n, step):
            g.add_dev(synth.rows(r0, min(step, n - r0)))
        g.finalize()
        g.nprobe = nprobe
        cent, off = g.get_centroids(), g.get_array("list_off")
        if cent0 is None:
            cent0, off0 = cent, off
        I = g.search_dev(xq_t, k)[1].cpu().numpy()
        xs = xq_t[:32].cpu().numpy()
        Dg, Ig = g.search(xs, k)
        o = OracleIVFPQR(d, nlist, M, M2) if M2 else O.make_index("ivf_pq", d, metric=O.METRIC_L2, nlist=nlist, M=M)
        o.set_state(g.get_state())
        o.nprobe = nprobe
        Do, Io = o.search(xs, k)
        del o
        res[case] = {
            "M": M, "M2": M2, "bytes_per_vector_stored": M + M2 + 8,
            "recall_at_10": float(np.mean([len(set(a) & set(b)) / k for a, b in zip(I, exact)])),
            "same_centroids_and_lists_as_PQ16": bool(np.array_equal(cent, cent0) and np.array_equal(off, off0)),
            "bit_exact_vs_oracle_32q": bool(np.array_equal(Dg, Do) and np.array_equal(Ig, Io)),
            "batch_ms_rounds": [], "scan_kernel_ms_rounds": [], "refine_ms_rounds": [],
        }
        shards[case] = g
        print(json.dumps({name: {case: res[case]}}), flush=True)

    for _ in range(rounds):
        for case, _, M2 in CASES:
            g = shards[case]
            res[case]["batch_ms_rounds"].append(timed(lambda: g.search_dev(xq_t, k)))
            g.profile(True)
            for _ in range(reps):
                g.search_dev(xq_t, k)
            torch.cuda.synchronize()
            if M2:
                res[case]["refine_ms_rounds"].append(g.get_param("refine_ms") / reps)
            scan_ms, _ = g.profile_read()
            g.profile(False)
            res[case]["scan_kernel_ms_rounds"].append(scan_ms / reps)
            res[case]["ndis"] = g.last_stats()["ndis"]

    for case, _, M2 in CASES:
        r = res[case]
        r.update({
            "batch_ms": float(np.median(r["batch_ms_rounds"])),
            "scan_kernel_ms": float(np.median(r["scan_kernel_ms_rounds"])),
            "scan_kernel_ms_min_max": [min(r["scan_kernel_ms_rounds"]), max(r["scan_kernel_ms_rounds"])],
            "qps": nq / float(np.median(r["batch_ms_rounds"])) * 1e3,
        })
        if M2:
            r["refine_ms"] = float(np.median(r["refine_ms_rounds"]))
            r["refine_ms_min_max"] = [min(r["refine_ms_rounds"]), max(r["refine_ms_rounds"])]
        else:
            del r["refine_ms_rounds"]
    del shards
    torch.cuda.empty_cache()
    return res


def main():
    d, n, nlist, nprobe, nq, k = 128, int(os.environ.get("PQR_BENCH_N", 10_000_000)), 4096, 32, 1000, 10
    rounds, reps = 3, 10
    out = {"card": card(), "setup": {"d": d, "n": n, "nlist": nlist, "nprobe": nprobe, "nq": nq, "k": k,
                                     "k_factor": 4, "rounds": rounds, "reps_per_round": reps}}
    for name, p in DATASETS.items():
        out[name] = run_dataset(name, p, d, n, nlist, nprobe, nq, k, rounds, reps)
    print(json.dumps(out, indent=1))


if __name__ == "__main__":
    main()
