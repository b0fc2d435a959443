#!/usr/bin/env python
"""IVF-PQ with 4-bit codes against 8-bit codes on one H100: the shuffle-lookup scan
(scan_pq4_kernel, table in registers) next to the 8-bit scans at equal bytes or equal lookups.

Shard: the bench generator at d = 128 (bench.py's defaults), 10M vectors, nlist 4096, nprobe 32,
1 000 device-resident queries, k = 10.  The coarse k-means runs with the same seed on the same rows
for every case, so every shard holds the same centroids and lists (checked and reported); only the
codes differ.  Cases:
  pq8_M32   the interleaved fused scan (the bench's kernel)        32 B per vector
  pq8_M16   scan_pq_kernel<16>                                     16 B per vector
  pq8_M64   scan_pq_kernel<64>                                     64 B per vector, 64 lookups
  pq4_M32   scan_pq4_kernel<32>                                    16 B per vector (= pq8_M16)
  pq4_M64   scan_pq4_kernel<64>                                    32 B per vector (= pq8_M32), 64 lookups (= pq8_M64)
All five shards stay resident and are timed in alternating rounds, so that the spread across rounds
is visible.  Per case:
  batch_ms         one search of the 1 000 queries (CUDA events, median over rounds)
  scan_kernel_ms   the list-scan launch alone (dfx_profile_*: bracketed by CUDA events; for pq8_M32
                   the fused table build + scan), median and [min, max] over rounds
  vectors_per_s    ndis over scan_kernel_ms;  lookups_per_s = ndis x M over it
  code_GBps        ndis x code bytes over scan_kernel_ms, and its fraction of 3.35 TB/s (H100 SXM
                   HBM3 data sheet); row_GBps adds the 4 B t-value and 4 B id every vector reads
  recall_at_10     against the exact top-10 of the GPU flat (L2) index over the same vectors
  bit_exact_vs_oracle_32q  a query sample against the oracle holding the same shard state
The card name and its power limit are read in the same run and recorded with the numbers."""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import kind_bench as kb  # noqa: E402
from distributed_faiss_b200 import engine  # noqa: E402
from oracle import oracle as O  # noqa: E402

HBM_BPS = 3.35e12
CASES = (("pq8_M32", 8, 32), ("pq8_M16", 8, 16), ("pq8_M64", 8, 64), ("pq4_M32", 4, 32), ("pq4_M64", 4, 64))


def main():
    d, n, nlist, nprobe, nq, k = 128, int(os.environ.get("PQ4_BENCH_N", 10_000_000)), 4096, 32, 1000, 10
    rounds, reps = 3, 10
    out = {"card": kb.card(), "setup": {"d": d, "n": n, "nlist": nlist, "nprobe": nprobe, "nq": nq, "k": k,
                                        "rounds": rounds, "reps_per_round": reps}}
    ds = kb.Dataset(d, n, nq, step=1_000_000)
    ds.exact(k)
    xs = ds.sample()

    cases, res = [], {}
    same_lists = kb.SameLists()
    for name, nbits, M in CASES:
        g = ds.fill(engine.GpuIndex(engine.KIND_IVF_PQ, d, engine.METRIC_L2, nlist=nlist, pq_m=M, pq_nbits=nbits),
                    nlist, nprobe)
        same = same_lists(g)
        o = O.make_index("ivf_pq", d, metric=O.METRIC_L2, nlist=nlist, M=M, nbits=nbits)
        res[name] = {
            "nbits": nbits, "M": M, "code_bytes_per_vector": M * nbits // 8,
            "recall_at_10": ds.recall(g, k),
            "same_centroids_and_lists_as_pq8_M32": same,
            "bit_exact_vs_oracle_32q": kb.same_arrays(g.search(xs, k), kb.mirror(o, g, nprobe).search(xs, k)),
            "batch_ms_rounds": [], "scan_kernel_ms_rounds": [],
        }
        del o
        cases.append((name, g, 0, False))
        print(json.dumps({name: res[name]}), flush=True)

    kb.time_rounds(cases, res, ds.xq, k, rounds, reps)
    for name, nbits, M in CASES:
        r = res[name]
        ndis, cb = r["ndis"], r["code_bytes_per_vector"]
        scan_s = r["scan_kernel_ms"] * 1e-3
        r.update({
            "vectors_per_s": ndis / scan_s, "lookups_per_s": ndis * M / scan_s,
            "code_GBps": ndis * cb / scan_s / 1e9, "code_fraction_of_hbm": ndis * cb / scan_s / HBM_BPS,
            "row_GBps": ndis * (cb + 8) / scan_s / 1e9, "row_fraction_of_hbm": ndis * (cb + 8) / scan_s / HBM_BPS,
        })
    out.update(res)
    out["pq4_M64_over_pq8_M64_lookups"] = res["pq4_M64"]["lookups_per_s"] / res["pq8_M64"]["lookups_per_s"]
    out["pq4_M32_over_pq8_M32_vectors"] = res["pq4_M32"]["vectors_per_s"] / res["pq8_M32"]["vectors_per_s"]
    print(json.dumps(out, indent=1))


if __name__ == "__main__":
    main()
