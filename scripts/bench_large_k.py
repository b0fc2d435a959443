#!/usr/bin/env python
"""IVF search at k > 1024 on one H100: every probed vector's composite written to its candidate row,
then one k-selection per query (dfx_search.cu), next to the k = 1024 path (per-warp queues).

Shards: the bench generator at d = 128 (bench.py's defaults), 10M vectors, nlist 4096, nprobe 32,
1 000 device-resident queries; IVF-PQ M = 32 (the interleaved block scan) and IVF-SQ8.
k = 1024 (the per-warp-queue path, the baseline), 1025, 2048 and 4096.  Per shard and k:
  batch_ms               one search of the 1 000 queries (CUDA events, median over rounds)
  kernels_us             torch.profiler, in a run of its own: device time per search of the list scan,
                         the final selection (select_cand_kernel; at k = 1024 the reduction of the
                         per-group partial results), the candidate offsets (k > 1024) and the rest
  cand_bytes_written     ndis x 8 B (k > 1024: one composite per scanned vector)
  cand_bytes_per_pass    ndis x 8 B: the selection reads the candidate rows once per radix pass and
                         once more to collect the k best
  bit_exact_vs_oracle_32q  32 queries against the oracle holding the same shard state
The card name and its power limit are read in the same run and recorded with the numbers."""
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import kind_bench as kb  # noqa: E402
from distributed_faiss_b200 import engine  # noqa: E402
from tests import oracle_sq8 as S  # noqa: E402

KS = (1024, 1025, 2048, 4096)


def kernel_breakdown(fn, reps):
    """device microseconds per call of fn, by kernel family"""
    from torch.profiler import ProfilerActivity, profile

    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            fn()
        torch.cuda.synchronize()
    fam = {"scan": 0.0, "select": 0.0, "cand_offsets": 0.0, "other": 0.0}
    for e in prof.key_averages():
        t = getattr(e, "device_time_total", None)
        if t is None:
            t = e.cuda_time_total
        if t <= 0:
            continue
        name = e.key
        if "cand_offsets" in name:
            fam["cand_offsets"] += t
        elif "scan_" in name and "kernel" in name:
            fam["scan"] += t
        elif "select_cand" in name or ("dfx_select_rows_kernel" in name and "ResultWriter" in name):
            fam["select"] += t
        else:
            fam["other"] += t
    return {k: v / reps for k, v in fam.items()}


def main():
    assert torch.cuda.is_available(), "bench_large_k measures the GPU: no CUDA device"
    d, n, nlist, nprobe, nq = 128, int(os.environ.get("LARGE_K_BENCH_N", 10_000_000)), 4096, 32, 1000
    rounds, reps = 3, 5
    out = {"card": kb.card(), "setup": {"d": d, "n": n, "nlist": nlist, "nprobe": nprobe, "nq": nq, "ks": KS,
                                        "rounds": rounds, "reps_per_round": reps}}
    ds = kb.Dataset(d, n, nq, step=1_000_000)
    xq_t, xs = ds.xq, ds.sample()

    for name, kind, M in (("ivf_pq_M32", engine.KIND_IVF_PQ, 32), ("ivf_sq8", engine.KIND_IVF_SQ8, 0)):
        g = ds.fill(engine.GpuIndex(kind, d, engine.METRIC_L2, nlist=nlist, pq_m=M), nlist, nprobe)
        o = kb.mirror(S.make_index(engine.KIND_NAMES[kind], d, metric=S.O.METRIC_L2, nlist=nlist, M=M), g, nprobe)
        lens = np.sort(np.diff(o.list_off))[::-1]
        res = {"candidate_row_bound": int(lens[:nprobe].sum())}
        for k in KS:
            bit_exact = kb.same_arrays(g.search(xs, k), o.search(xs, k))
            g.search_dev(xq_t, k)
            ndis = g.last_stats()["ndis"]
            batch = [kb.timed(lambda: g.search_dev(xq_t, k), iters=reps) for _ in range(rounds)]
            r = {
                "bit_exact_vs_oracle_32q": bit_exact,
                "ndis": ndis,
                "batch_ms": float(np.median(batch)), "batch_ms_rounds": batch,
                "kernels_us": kernel_breakdown(lambda: g.search_dev(xq_t, k), reps),
                "cand_bytes_written": ndis * 8 if k > 1024 else 0,
                "cand_bytes_per_pass": ndis * 8 if k > 1024 else 0,
                "workspace_bytes": g.get_param("workspace_bytes"),
            }
            res[f"k{k}"] = r
            print(json.dumps({name: {f"k{k}": r}}), flush=True)
        out[name] = res
        del g, o
        torch.cuda.empty_cache()
    print(json.dumps(out, indent=1))


if __name__ == "__main__":
    main()
