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
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import kind_bench as kb  # noqa: E402
from distributed_faiss_b200 import engine  # noqa: E402
from oracle import oracle as O  # noqa: E402
from tests import oracle_sq8  # noqa: E402


def main():
    out = {"card": kb.card()}
    # ---- C1
    rs = np.random.RandomState(0)
    xb = rs.rand(100_000, 128).astype(np.float32)
    xq = rs.rand(1000, 128).astype(np.float32)
    g = engine.GpuIndex(engine.KIND_FLAT, 128, engine.METRIC_INNER_PRODUCT)
    g.add(xb)
    xq_t = torch.from_numpy(xq).cuda()
    ms = kb.timed(lambda: g.search_dev(xq_t, 10))
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
    # ---- C2 / C4 on the bench generator; both C4 shards share one dataset and its exact top-10
    c2 = kb.Dataset(128, 10_000_000, 1000, step=500_000, seed=99)
    c4 = kb.Dataset(768, 2_000_000, 1000, step=500_000, seed=99, r=32)
    for name, kind, okind, ds, nlist in (("C2_ivf_simple_10M", engine.KIND_IVF_FLAT, "ivf_flat", c2, 4096),
                                         ("C4_ivfsq_d768_2M", engine.KIND_IVF_SQ16, "ivf_sq", c4, 2048),
                                         ("C4_ivfsq8_d768_2M", engine.KIND_IVF_SQ8, "ivf_sq8", c4, 2048)):
        d = ds.d
        g = ds.fill(engine.GpuIndex(kind, d, engine.METRIC_L2, nlist=nlist), nlist, 32)
        ms, scan_ms, _, ndis = kb.measure(g, ds.xq, 10, reps=5)
        row_bytes = {engine.KIND_IVF_FLAT: 4 * d, engine.KIND_IVF_SQ16: 2 * d, engine.KIND_IVF_SQ8: d}[kind]
        xs = ds.sample(64)
        D, I = g.search(xs, 10)
        o = kb.mirror(oracle_sq8.make_index(okind, d, metric=O.METRIC_L2, nlist=nlist), g, 32)
        bit_exact = kb.same_arrays((D, I), o.search(xs, 10))
        self_hit = float((I[:, 0] == ds.rows[:64].cpu().numpy()).mean())
        out[name] = {"ms": ms, "qps": 1000 / ms * 1e3, "ndis": ndis,
                     "scan_GBps_algorithmic": ndis * row_bytes / ms / 1e6, "scan_kernel_ms": scan_ms, "scan_kernel_GBps_algorithmic": ndis * row_bytes / scan_ms / 1e6,
                     "bit_exact_vs_oracle_64q": bit_exact, "top1_is_source_row": self_hit}
        if d == 768:
            out[name]["recall_at_10"] = ds.recall(g, 10)
        del g
    print(json.dumps(out, indent=1))


if __name__ == "__main__":
    main()
