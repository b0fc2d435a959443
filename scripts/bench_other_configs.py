#!/usr/bin/env python
"""Timing of the other BASELINE.json configurations on one H100 (they are parity-test cases,
not bench lines; this records where their kernels stand):
  C1 flat d=128, 100k vectors, 1k queries          (configs[0])
  C2 ivf_simple d=128, 10M vectors, nlist 4096, nprobe 32   (configs[1])
  C4 ivfsq d=768, 2M-vector slice of one shard, nlist 2048, nprobe 32, 1k queries (configs[3], scaled)
  C4 the same shard as IVF-SQ8 ("IVF2048,SQ8"): same generator slice and training seed, so both
     shards hold the same centroids and lists; d bytes per vector instead of 2 d
Each case: device-resident queries, CUDA events, 3 warm-ups, plus a bit-exact check of a query
sample against the oracle holding the same shard state.  The C4 lines also report recall@10
against the exact top-10 of the GPU flat (L2) index over the same 2M vectors.  The card name and
its power limit are recorded with the numbers."""
import subprocess
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from distributed_faiss_b200 import engine  # noqa: E402
from oracle import oracle as O  # noqa: E402
from tests import oracle_sq8  # noqa: E402


def timed(fn, iters=10, warm=3):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def card():
    """name and power limit of the card the numbers were taken on (a read-only query)"""
    try:
        q = subprocess.run(["nvidia-smi", "-i", str(torch.cuda.current_device()), "--query-gpu=power.limit",
                            "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = "unknown"
    return {"name": torch.cuda.get_device_name(), "power_limit": q}


def main():
    out = {"card": card()}
    # ---- C1
    rs = np.random.RandomState(0)
    xb = rs.rand(100_000, 128).astype(np.float32)
    xq = rs.rand(1000, 128).astype(np.float32)
    g = engine.GpuIndex(engine.KIND_FLAT, 128, engine.METRIC_INNER_PRODUCT)
    g.add(xb)
    xq_t = torch.from_numpy(xq).cuda()
    ms = timed(lambda: g.search_dev(xq_t, 10))
    D, I = g.search(xq, 10)
    o = O.make_index("flat", 128, metric=O.METRIC_IP)
    o.add(xb)
    t0 = time.perf_counter()
    Do, Io = o.search(xq, 10)
    cpu_s = time.perf_counter() - t0
    out["C1_flat_100k_1k"] = {"ms": ms, "qps": 1000 / ms * 1e3, "tflops_algorithmic": 2 * 1000 * 1e5 * 128 / ms / 1e9,
                              "bit_exact_vs_oracle": bool(np.array_equal(D, Do) and np.array_equal(I, Io)),
                              "cpu_oracle_qps": 1000 / cpu_s, "cpu_cores": O.num_threads()}
    del g
    # ---- C2 / C4 on the bench generator
    exact = {}
    for name, kind, okind, d, n, nlist, rank in (("C2_ivf_simple_10M", engine.KIND_IVF_FLAT, "ivf_flat", 128, 10_000_000, 4096, 16),
                                                 ("C4_ivfsq_d768_2M", engine.KIND_IVF_SQ16, "ivf_sq", 768, 2_000_000, 2048, 32),
                                                 ("C4_ivfsq8_d768_2M", engine.KIND_IVF_SQ8, "ivf_sq8", 768, 2_000_000, 2048, 32)):
        synth = engine.Synth(99, d, rank, 1, 1.0, 0.02, ngroups=n // 10, eps=0.01, delta=0.1)
        g = engine.GpuIndex(kind, d, engine.METRIC_L2, nlist=nlist)
        g.set_param("kmeans_niter", 10)
        g.set_param("max_points_per_centroid", 64)
        g.train_dev(synth.rows(0, 64 * nlist))
        step = 500_000
        for r0 in range(0, n, step):
            g.add_dev(synth.rows(r0, min(step, n - r0)))
        g.finalize()
        g.nprobe = 32
        rows = torch.randint(0, n, (1000,), dtype=torch.int64, generator=torch.Generator().manual_seed(1)).cuda()
        xq_t = synth.rows(0, 1000, rows_t=rows, noise_stream=7)
        ms = timed(lambda: g.search_dev(xq_t, 10))
        g.profile(True)  # the list-scan kernel alone, bracketed by CUDA events
        for _ in range(5):
            g.search_dev(xq_t, 10)
        torch.cuda.synchronize()
        scan_ms, launches = g.profile_read()
        g.profile(False)
        scan_ms /= 5
        st = g.last_stats()
        row_bytes = {engine.KIND_IVF_FLAT: 4 * d, engine.KIND_IVF_SQ16: 2 * d, engine.KIND_IVF_SQ8: d}[kind]
        D, I = g.search(xq_t[:64].cpu().numpy(), 10)
        o = oracle_sq8.make_index(okind, d, metric=O.METRIC_L2, nlist=nlist)
        o.set_state(g.get_state())
        o.nprobe = 32
        Do, Io = o.search(xq_t[:64].cpu().numpy(), 10)
        self_hit = float((I[:, 0] == rows[:64].cpu().numpy()).mean())
        out[name] = {"ms": ms, "qps": 1000 / ms * 1e3, "ndis": st["ndis"], "scan_GBps_algorithmic": st["ndis"] * row_bytes / ms / 1e6,
                     "scan_kernel_ms": scan_ms, "scan_kernel_GBps_algorithmic": st["ndis"] * row_bytes / scan_ms / 1e6,
                     "bit_exact_vs_oracle_64q": bool(np.array_equal(D, Do) and np.array_equal(I, Io)), "top1_is_source_row": self_hit}
        if d == 768:
            if "C4" not in exact:  # exact top-10 of the same 2M vectors, GPU flat L2 index
                flat = engine.GpuIndex(engine.KIND_FLAT, d, engine.METRIC_L2)
                flat.reserve(n)
                for r0 in range(0, n, step):
                    flat.add_dev(synth.rows(r0, min(step, n - r0)))
                exact["C4"] = flat.search_dev(xq_t, 10)[1].cpu().numpy()
                del flat
            Ia = g.search_dev(xq_t, 10)[1].cpu().numpy()
            out[name]["recall_at_10"] = float(np.mean([len(set(a) & set(b)) / 10 for a, b in zip(Ia, exact["C4"])]))
        del g
    print(json.dumps(out, indent=1))


if __name__ == "__main__":
    main()
