#!/usr/bin/env python
"""IVF-PQ at M = 48, 64, 96 and 128 on one H100: the row-major scan at M <= 64 (scan_pq_kernel<0> for
M = 48, whose 16-byte dsub keeps d = 768, and scan_pq_kernel<64>) and the wide-code scan above it
(scan_pq_wide_kernel, table built in shared memory).

Shard: synthetic d = 768 (the bench generator), 2M vectors, nlist 2048, 1 000 queries, nprobe 32,
k = 10.  The coarse k-means runs with the same seed on the same rows for every M, so the shards
hold the same centroids and lists (checked and reported); only the codes differ.  All four shards
stay resident and are timed in alternating rounds, so that the spread across rounds is visible.
Per M:
  batch_ms         one search of the 1 000 device-resident queries (CUDA events, median over rounds)
  scan_kernel_ms   the list-scan launch alone (dfx_profile_*: the table + |q - c|^2 preparation and
                   the scan, bracketed by CUDA events), median and [min, max] over rounds
  lookups_per_s    ndis x M table lookups over scan_kernel_ms
  code_GBps        ndis x M code bytes over scan_kernel_ms
  recall_at_10     against the exact top-10 of the GPU flat (L2) index over the same 2M vectors
  bit_exact_vs_oracle_32q  a query sample against the oracle holding the same shard state
The card name and its power limit are recorded with the numbers."""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import kind_bench as kb  # noqa: E402
from distributed_faiss_b200 import engine  # noqa: E402
from oracle import oracle as O  # noqa: E402


def main():
    d, n, nlist, nprobe, nq, k = 768, 2_000_000, 2048, 32, 1000, 10
    rounds, reps = 3, 10
    out = {"card": kb.card(), "setup": {"d": d, "n": n, "nlist": nlist, "nprobe": nprobe, "nq": nq, "k": k,
                                        "rounds": rounds, "reps_per_round": reps}}
    ds = kb.Dataset(d, n, nq, step=500_000, seed=99, r=32)
    ds.exact(k)
    xs = ds.sample()

    cases, res = [], {}
    same_lists = kb.SameLists()
    for M in (48, 64, 96, 128):
        name = f"M{M}"
        g = ds.fill(engine.GpuIndex(engine.KIND_IVF_PQ, d, engine.METRIC_L2, nlist=nlist, pq_m=M), nlist, nprobe)
        same = same_lists(g)
        o = O.make_index("ivf_pq", d, metric=O.METRIC_L2, nlist=nlist, M=M)
        res[name] = {
            "recall_at_10": ds.recall(g, k), "same_centroids_and_lists_as_M48": same,
            "bit_exact_vs_oracle_32q": kb.same_arrays(g.search(xs, k), kb.mirror(o, g, nprobe).search(xs, k)),
        }
        del o
        cases.append((name, g, 0, False))
        print(json.dumps({name: res[name]}), flush=True)

    kb.time_rounds(cases, res, ds.xq, k, rounds, reps)
    for name, _, _, _ in cases:
        r = res[name]
        lookups_per_s = r["ndis"] * int(name[1:]) / (r["scan_kernel_ms"] * 1e-3)
        r.update({"lookups_per_s": lookups_per_s, "code_GBps": lookups_per_s / 1e9})
    out.update(res)
    print(json.dumps(out, indent=1))


if __name__ == "__main__":
    main()
