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

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))
from bench_other_configs import card, timed  # noqa: E402
from distributed_faiss_b200 import engine  # noqa: E402
from oracle import oracle as O  # noqa: E402
from tests.oracle_pq_fs import OracleIVFPQFastScan  # noqa: E402

HBM_BPS = 3.35e12
CASES = (("fs_M32", "fs", 32), ("pq4_M32", "pq4", 32), ("fs_M64", "fs", 64), ("pq4_M64", "pq4", 64))


def main():
    d, n, nlist, nprobe, nq, k = 128, int(os.environ.get("FS_BENCH_N", 10_000_000)), 4096, 32, 1000, 10
    rounds, reps = 3, 10
    step = 1_000_000
    out = {"card": card(), "setup": {"d": d, "n": n, "nlist": nlist, "nprobe": nprobe, "nq": nq, "k": k,
                                     "rounds": rounds, "reps_per_round": reps}}
    synth = engine.Synth(1234, d, 16, 1, 1.0, 0.02, ngroups=max(1, n // 10), eps=0.01, delta=0.1)
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
    for name, what, M in CASES:
        kind = engine.KIND_IVF_PQ_FS if what == "fs" else engine.KIND_IVF_PQ
        g = engine.GpuIndex(kind, d, engine.METRIC_L2, nlist=nlist, pq_m=M, pq_nbits=4)
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
        if what == "fs":
            o = OracleIVFPQFastScan(d, nlist, M)
        else:
            o = O.make_index("ivf_pq", d, metric=O.METRIC_L2, nlist=nlist, M=M, nbits=4)
        o.set_state(g.get_state())
        o.nprobe = nprobe
        Do, Io = o.search(xs, k)
        del o
        row_bytes = M // 2 + 4 + (4 if what == "pq4" else 0)
        res[name] = {
            "M": M, "row_bytes_per_vector": row_bytes,
            "recall_at_10": float(np.mean([len(set(a) & set(b)) / k for a, b in zip(I, exact)])),
            "same_centroids_and_lists_as_fs_M32": bool(np.array_equal(cent, cent0) and np.array_equal(off, off0)),
            "bit_exact_vs_oracle_32q": bool(np.array_equal(Dg, Do) and np.array_equal(Ig, Io)),
            "batch_ms_rounds": [], "scan_kernel_ms_rounds": [],
        }
        shards[name] = g
        print(json.dumps({name: res[name]}), flush=True)

    for _ in range(rounds):
        for name, _, _ in CASES:
            g = shards[name]
            res[name]["batch_ms_rounds"].append(timed(lambda: g.search_dev(xq_t, k)))
            g.profile(True)
            for _ in range(reps):
                g.search_dev(xq_t, k)
            torch.cuda.synchronize()
            scan_ms, _ = g.profile_read()
            g.profile(False)
            res[name]["scan_kernel_ms_rounds"].append(scan_ms / reps)
            res[name]["ndis"] = g.last_stats()["ndis"]

    for name, _, M in CASES:
        r = res[name]
        scan_ms = float(np.median(r["scan_kernel_ms_rounds"]))
        ndis, rb = r["ndis"], r["row_bytes_per_vector"]
        scan_s = scan_ms * 1e-3
        r.update({
            "batch_ms": float(np.median(r["batch_ms_rounds"])), "scan_kernel_ms": scan_ms,
            "scan_kernel_ms_min_max": [min(r["scan_kernel_ms_rounds"]), max(r["scan_kernel_ms_rounds"])],
            "qps": nq / float(np.median(r["batch_ms_rounds"])) * 1e3,
            "vectors_per_s": ndis / scan_s, "lookups_per_s": ndis * M / scan_s,
            "row_GBps": ndis * rb / scan_s / 1e9, "row_fraction_of_hbm": ndis * rb / scan_s / HBM_BPS,
        })
    out.update(res)
    out["fs_M32_over_pq4_M32_vectors"] = res["fs_M32"]["vectors_per_s"] / res["pq4_M32"]["vectors_per_s"]
    out["fs_M64_over_pq4_M64_vectors"] = res["fs_M64"]["vectors_per_s"] / res["pq4_M64"]["vectors_per_s"]
    print(json.dumps(out, indent=1))


if __name__ == "__main__":
    main()
