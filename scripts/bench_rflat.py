#!/usr/bin/env python
"""Flat refinement ("IVF{n},<codec>,RFlat": the codec's search for k' = k * k_factor candidates, re-ranked
on the stored fp32 rows by rflat_refine_kernel) against the plain codec shards and IVF-Flat on one H100.

Shards: d = 128, nlist 4096, nprobe 32, 1 000 device-resident queries, k = 10, on the two datasets of
scripts/kind_bench.py (RFLAT_BENCH_DATASETS picks one), RFLAT_BENCH_N (default 10M) vectors each:
  bench      the bench generator (bench.py's defaults: near-duplicate groups, low intrinsic dimension)
  clustered  the same generator as plain clustered data: 10 000 Gaussian clusters in 16 dimensions,
             no near-duplicate groups, per-row noise in all 128
The coarse k-means runs with the same seed on the same rows for every shard, so every shard of one
dataset holds the same centroids and lists (checked and reported).  Cases, per codec FS16
("PQ16x4fs"), FS32 ("PQ32x4fs") and PQ16:
  <codec>            the plain shard (the refined shard's lists imported into a shard without refinement)
  <codec>,RFlat x4   k' = 40 candidates re-ranked      <codec>,RFlat x10   k' = 100
and IVF-Flat on the same centroids, the exact ceiling at this nprobe.  The shards of a dataset stay
resident and are timed in alternating rounds.  Per case:
  batch_ms         one search of the 1 000 queries (CUDA events, median over rounds)
  scan_kernel_ms   the first-stage list scan (dfx_profile_*: bracketed by CUDA events)
  refine_ms        the re-ranking kernel + its final selection (dfx_get_param "refine_ms")
  gather_bytes     nq * k' * 4 d, the rows the re-ranking reads; gather_share_of_hbm_peak is
                   gather_bytes / refine_ms over the data sheet's 3.35 TB/s -- refine_ms includes the
                   selection, so this is a lower bound for the kernel alone
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
from tests.oracle_rflat import make_rflat  # noqa: E402

CODECS = (("FS16", engine.KIND_IVF_PQ_FS, "ivf_pq_fs", 16, 4), ("FS32", engine.KIND_IVF_PQ_FS, "ivf_pq_fs", 32, 4),
          ("PQ16", engine.KIND_IVF_PQ, "ivf_pq", 16, 8))
K_FACTORS = (4, 10)
HBM_PEAK = 3.35e12  # B/s, H100 SXM data sheet


def plain_copy(g, kind, d, nlist, M, nbits):
    """the same centroids, codebooks and lists in a shard without the refinement"""
    p = engine.GpuIndex(kind, d, engine.METRIC_L2, nlist=nlist, pq_m=M, pq_nbits=nbits)
    p.set_state({key: g.get_array(key) for key in ("centroids", "codebooks", "list_off", "ids", "codes")})
    return p


def run_dataset(name, p, d, n, nlist, nprobe, nq, k, rounds, reps):
    ds = kb.Dataset(d, n, nq, step=1_000_000, **p)
    xs = ds.sample()
    ds.exact(k)

    cases, res = [], {}   # (case name, shard, k_factor or 0, whether it re-ranks)
    same_lists = kb.SameLists()
    ivf = ds.fill(engine.GpuIndex(engine.KIND_IVF_FLAT, d, engine.METRIC_L2, nlist=nlist), nlist, nprobe, reserve=True)
    same_lists(ivf)
    cases.append(("IVF-Flat", ivf, 0, False))
    res["IVF-Flat"] = {"bytes_per_vector_stored": 4 * d + 4, "recall_at_10": ds.recall(ivf, k)}
    for codec, kind, kname, M, nbits in CODECS:
        g = engine.GpuIndex(kind, d, engine.METRIC_L2, nlist=nlist, pq_m=M, pq_nbits=nbits, refine_flat=True)
        ds.fill(g, nlist, nprobe, reserve=True)
        same = same_lists(g)
        plain = plain_copy(g, kind, d, nlist, M, nbits)
        plain.nprobe = nprobe
        row = (M if nbits == 8 else M // 2) + (8 if nbits == 8 else 4)   # code (+ t-value) + id
        cases.append((codec, plain, 0, False))
        res[codec] = {"bytes_per_vector_stored": row, "recall_at_10": ds.recall(plain, k),
                      "same_centroids_and_lists_as_IVF_Flat": same}
        o = kb.mirror(make_rflat(kname, d, nlist, M), g, nprobe)
        for kf in K_FACTORS:
            case = f"{codec},RFlat x{kf}"
            g.set_param("k_factor", kf)
            o.k_factor = float(kf)
            bit_exact = kb.same_arrays(g.search(xs, k), o.search(xs, k))
            cases.append((case, g, kf, True))
            res[case] = {"bytes_per_vector_stored": row + 4 * d, "k_first_stage": k * kf,
                         "recall_at_10": ds.recall(g, k), "same_centroids_and_lists_as_IVF_Flat": same,
                         "bit_exact_vs_oracle_32q": bit_exact, "gather_bytes": nq * k * kf * 4 * d}
        del o
        for case in [c for c, _, _, _ in cases if c.startswith(codec)]:
            print(json.dumps({name: {case: res[case]}}), flush=True)

    kb.time_rounds(cases, res, ds.xq, k, rounds, reps)
    for case, _, kf, _ in cases:
        if kf:
            r = res[case]
            r["gather_share_of_hbm_peak"] = r["gather_bytes"] / (r["refine_ms"] * 1e-3) / HBM_PEAK
    del cases
    torch.cuda.empty_cache()
    return res


def main():
    d, n, nlist, nprobe, nq, k = 128, int(os.environ.get("RFLAT_BENCH_N", 10_000_000)), 4096, 32, 1000, 10
    rounds, reps = 3, 10
    out = {"card": kb.card(), "setup": {"d": d, "n": n, "nlist": nlist, "nprobe": nprobe, "nq": nq, "k": k,
                                        "k_factors": K_FACTORS, "rounds": rounds, "reps_per_round": reps}}
    for name in os.environ.get("RFLAT_BENCH_DATASETS", ",".join(kb.DATASETS)).split(","):
        out[name] = run_dataset(name, kb.DATASETS[name], d, n, nlist, nprobe, nq, k, rounds, reps)
    print(json.dumps(out, indent=1))


if __name__ == "__main__":
    main()
