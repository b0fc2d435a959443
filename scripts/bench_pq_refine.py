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

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import kind_bench as kb  # noqa: E402
from distributed_faiss_b200 import engine  # noqa: E402
from oracle import oracle as O  # noqa: E402
from tests.oracle_pqr import OracleIVFPQR  # noqa: E402

CASES = (("PQ16", 16, 0), ("PQ16+16", 16, 16), ("PQ32", 32, 0))


def run_dataset(name, p, d, n, nlist, nprobe, nq, k, rounds, reps):
    ds = kb.Dataset(d, n, nq, step=1_000_000, **p)
    ds.exact(k)
    xs = ds.sample()

    cases, res = [], {}
    same_lists = kb.SameLists()
    for case, M, M2 in CASES:
        kind = engine.KIND_IVF_PQR if M2 else engine.KIND_IVF_PQ
        g = ds.fill(engine.GpuIndex(kind, d, engine.METRIC_L2, nlist=nlist, pq_m=M, pq_nbits=8, refine_m=M2),
                    nlist, nprobe)
        same = same_lists(g)
        o = OracleIVFPQR(d, nlist, M, M2) if M2 else O.make_index("ivf_pq", d, metric=O.METRIC_L2, nlist=nlist, M=M)
        res[case] = {
            "M": M, "M2": M2, "bytes_per_vector_stored": M + M2 + 8,
            "recall_at_10": ds.recall(g, k),
            "same_centroids_and_lists_as_PQ16": same,
            "bit_exact_vs_oracle_32q": kb.same_arrays(g.search(xs, k), kb.mirror(o, g, nprobe).search(xs, k)),
            "batch_ms_rounds": [], "scan_kernel_ms_rounds": [], "refine_ms_rounds": [],
        }
        del o
        cases.append((case, g, 0, bool(M2)))
        print(json.dumps({name: {case: res[case]}}), flush=True)

    kb.time_rounds(cases, res, ds.xq, k, rounds, reps)
    del cases
    torch.cuda.empty_cache()
    return res


def main():
    d, n, nlist, nprobe, nq, k = 128, int(os.environ.get("PQR_BENCH_N", 10_000_000)), 4096, 32, 1000, 10
    rounds, reps = 3, 10
    out = {"card": kb.card(), "setup": {"d": d, "n": n, "nlist": nlist, "nprobe": nprobe, "nq": nq, "k": k,
                                        "k_factor": 4, "rounds": rounds, "reps_per_round": reps}}
    for name, p in kb.DATASETS.items():
        out[name] = run_dataset(name, p, d, n, nlist, nprobe, nq, k, rounds, reps)
    print(json.dumps(out, indent=1))


if __name__ == "__main__":
    main()
