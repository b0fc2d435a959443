#!/usr/bin/env python
"""Device time of the coarse quantizer's decide stage (dfx_tc.cu, DESIGN.md §4.1 item 4) per
search of 4096 queries, d = 128, on IVF-Flat shards with one vector per list (as
tests/test_tc_decide.py builds them), at each nlist, nprobe and screening precision.

The decide stage is every kernel between the screening and the list scan: the group selection
(`topg_collect_kernel`, or the radix select over the group minima), the warp-per-row decide kernel
and the exact fallback (`tc_exact_rows_kernel`).  Their device times come from torch.profiler over
ITERS searches and are summed per search.  `rerank2_kernel` is matched too, so that a build from
before it was folded into `decide_rows_kernel` can be timed by the same script; to compare two
builds, run the script on each in turn, alternating, and compare the medians.

The nlist values cover each source of a row's groups (one level in the kernel at 1024 and 3200
lists, given by the radix select at 2048, two levels at 65 536); nprobe 32 keeps G = 40 groups at
3200 and 65 536 lists, which the radix select gives too.  `ids_sha` hashes the ids of the first
search, which are its probe keys: it must not change between builds.  One JSON line per case.
    python scripts/bench_decide.py
"""
import hashlib
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import kind_bench  # noqa: E402
from distributed_faiss_b200 import engine  # noqa: E402

NQ, D, ITERS = 4096, 128, 20
NLISTS, NPROBES, MODES = (1024, 2048, 3200, 65536), (8, 32), ((1, "fast"), (2, "precise"))


def is_decide(name):
    if "dfx_select_rows_kernel" in name:
        return "ColsLoader" in name  # the radix select over group minima, not the list scan's
    return any(k in name for k in ("topg_collect_kernel", "decide_rows_kernel", "rerank2_kernel",
                                   "tc_exact_rows_kernel"))


def shard(nlist, rs):
    cent = rs.randn(nlist, D).astype(np.float32)
    g = engine.GpuIndex(engine.KIND_IVF_FLAT, D, engine.METRIC_L2, nlist=nlist)
    g.set_state({"centroids": cent, "list_off": np.arange(nlist + 1, dtype=np.int64),
                 "ids": np.arange(nlist, dtype=np.int64), "vecs": cent.copy()})
    xq = cent[rs.randint(0, nlist, NQ)] + 0.1 * rs.randn(NQ, D)
    return g, torch.from_numpy(xq.astype(np.float32)).cuda()


def decide_us(g, xq, nprobe):
    from torch.profiler import ProfilerActivity, profile

    for _ in range(3):
        g.search_dev(xq, nprobe)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(ITERS):
            g.search_dev(xq, nprobe)
        torch.cuda.synchronize()
    kernels = {}
    for ev in prof.key_averages():
        if ev.device_time_total > 0 and is_decide(ev.key):
            name = ev.key.split("(")[0].replace("void ", "")
            kernels[name] = {"launches_per_search": ev.count / ITERS, "us_per_search": ev.device_time_total / ITERS}
    return sum(k["us_per_search"] for k in kernels.values()), kernels


def main():
    torch.cuda.set_device(0)
    card = kind_bench.card()
    for nlist in NLISTS:
        g, xq = shard(nlist, np.random.RandomState(nlist))
        for nprobe in NPROBES:
            g.nprobe = nprobe
            for mode, name in MODES:
                g.set_param("tc_screen_mode", mode)
                _, ids = g.search_dev(xq, nprobe)
                sha = hashlib.sha256(ids.cpu().numpy().tobytes()).hexdigest()[:16]
                total, kernels = decide_us(g, xq, nprobe)
                print(json.dumps({"nlist": nlist, "nprobe": nprobe, "mode": name, "decide_us": round(total, 2),
                                  "ids_sha": sha, "kernels": kernels, "card": card}), flush=True)


if __name__ == "__main__":
    main()
