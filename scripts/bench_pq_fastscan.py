#!/usr/bin/env python
"""IVF-PQ FastScan ("IVF{n},PQ{M}x4fs": 4-bit codes of the raw vectors, u8 quantized tables, integer
sums; pq_fs_lut_kernel + scan_pq_fs_kernel) against 4-bit knnlm IVF-PQ (residual codes, fp32 tables;
pq_prep_kernel + scan_pq4_kernel) on one H100, at the same M.

Shard: the bench generator at d = 128 (bench.py's defaults), 10M vectors, nlist 4096, nprobe 32,
1 000 device-resident queries, k = 10.  The coarse k-means runs with the same seed on the same rows
for every case, so every shard holds the same centroids and lists (checked and reported); only the
codes differ.  Cases:
  fs_M32    scan_pq_fs_kernel<32>   16 B code + 4 B id per vector
  pq4_M32   scan_pq4_kernel<32>     16 B code + 4 B t-value + 4 B id
  fs_M64    scan_pq_fs_kernel<64>   32 B code + 4 B id
  pq4_M64   scan_pq4_kernel<64>     32 B code + 4 B t-value + 4 B id
All four shards stay resident and are timed in alternating rounds, so that the spread across rounds
is visible.  Per case:
  batch_ms         one search of the 1 000 queries (CUDA events, median over rounds)
  scan_kernel_ms   the table kernel + list-scan launch (dfx_profile_*: bracketed by CUDA events),
                   median and [min, max] over rounds
  vectors_per_s    ndis over scan_kernel_ms;  lookups_per_s = ndis x M over it
  row_GBps         ndis x row bytes (codes, id, and the t-value of pq4) over scan_kernel_ms, and its
                   fraction of 3.35 TB/s (H100 SXM HBM3 data sheet)
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
from tests.oracle_pq_fs import OracleIVFPQFastScan  # noqa: E402

HBM_BPS = 3.35e12
CASES = (("fs_M32", "fs", 32), ("pq4_M32", "pq4", 32), ("fs_M64", "fs", 64), ("pq4_M64", "pq4", 64))


def main():
    d, n, nlist, nprobe, nq, k = 128, int(os.environ.get("FS_BENCH_N", 10_000_000)), 4096, 32, 1000, 10
    rounds, reps = 3, 10
    out = {"card": kb.card(), "setup": {"d": d, "n": n, "nlist": nlist, "nprobe": nprobe, "nq": nq, "k": k,
                                        "rounds": rounds, "reps_per_round": reps}}
    ds = kb.Dataset(d, n, nq, step=1_000_000)
    ds.exact(k)
    xs = ds.sample()

    cases, res = [], {}
    same_lists = kb.SameLists()
    for name, what, M in CASES:
        kind = engine.KIND_IVF_PQ_FS if what == "fs" else engine.KIND_IVF_PQ
        g = ds.fill(engine.GpuIndex(kind, d, engine.METRIC_L2, nlist=nlist, pq_m=M, pq_nbits=4), nlist, nprobe)
        same = same_lists(g)
        if what == "fs":
            o = OracleIVFPQFastScan(d, nlist, M)
        else:
            o = O.make_index("ivf_pq", d, metric=O.METRIC_L2, nlist=nlist, M=M, nbits=4)
        row_bytes = M // 2 + 4 + (4 if what == "pq4" else 0)
        res[name] = {
            "M": M, "row_bytes_per_vector": row_bytes,
            "recall_at_10": ds.recall(g, k),
            "same_centroids_and_lists_as_fs_M32": same,
            "bit_exact_vs_oracle_32q": kb.same_arrays(g.search(xs, k), kb.mirror(o, g, nprobe).search(xs, k)),
            "batch_ms_rounds": [], "scan_kernel_ms_rounds": [],
        }
        del o
        cases.append((name, g, 0, False))
        print(json.dumps({name: res[name]}), flush=True)

    kb.time_rounds(cases, res, ds.xq, k, rounds, reps)
    for name, _, M in CASES:
        r = res[name]
        ndis, rb = r["ndis"], r["row_bytes_per_vector"]
        scan_s = r["scan_kernel_ms"] * 1e-3
        r.update({
            "vectors_per_s": ndis / scan_s, "lookups_per_s": ndis * M / scan_s,
            "row_GBps": ndis * rb / scan_s / 1e9, "row_fraction_of_hbm": ndis * rb / scan_s / HBM_BPS,
        })
    out.update(res)
    out["fs_M32_over_pq4_M32_vectors"] = res["fs_M32"]["vectors_per_s"] / res["pq4_M32"]["vectors_per_s"]
    out["fs_M64_over_pq4_M64_vectors"] = res["fs_M64"]["vectors_per_s"] / res["pq4_M64"]["vectors_per_s"]
    print(json.dumps(out, indent=1))


if __name__ == "__main__":
    main()
