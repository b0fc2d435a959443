"""The steps the per-kind benchmark scripts share: the card the numbers are taken on, CUDA-event
timing, the bench generator's rows and queries with their exact top-k, the build of a shard, the
checks against the oracle and against the first shard, and the timed rounds over resident shards.

Add no search to a step and do not reorder its searches: the coarse quantizer's AUTO precision
(DESIGN.md §4.1 item 6) switches on the rows a shard has seen, so an extra or reordered warm-up
search can move a timed window from PRECISE to FAST, which changes its time but not its results."""
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
from distributed_faiss_b200 import engine  # noqa: E402

# The generator parameters of the two datasets of bench_pq_refine.py and bench_rflat.py, as overrides
# of Dataset's defaults (bench.py's generator)
DATASETS = {
    "bench": {},
    "clustered": dict(nclusters=10_000, sigma_q=0.05, eps=0.3, delta=0.0, groups_per=0),
}


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


class Dataset:
    """n rows of the bench generator (engine.Synth) at dimension d, added to a shard `step` rows at a
    time, and nq device-resident queries: rows drawn with torch seed 1 (`rows`), regenerated with the
    query noise of stream 7 (`xq`).  groups_per rows share a near-duplicate group (0: no groups)."""

    def __init__(self, d, n, nq, step, seed=1234, r=16, nclusters=1, sigma=1.0, sigma_q=0.02, eps=0.01, delta=0.1,
                 groups_per=10):
        ngroups = max(1, n // groups_per) if groups_per else 0
        if ngroups:
            ngroups = max(nclusters, ngroups // nclusters * nclusters)
        self.d, self.n, self.step = d, n, step
        self.synth = engine.Synth(seed, d, r, nclusters, sigma, sigma_q, ngroups=ngroups, eps=eps, delta=delta)
        self.rows = torch.randint(0, n, (nq,), dtype=torch.int64, generator=torch.Generator().manual_seed(1)).cuda()
        self.xq = self.synth.rows(0, nq, rows_t=self.rows, noise_stream=7)
        self._exact = {}

    def sample(self, m=32):
        """the first m queries on the host: the sample checked against the oracle"""
        return self.xq[:m].cpu().numpy()

    def add(self, g):
        for r0 in range(0, self.n, self.step):
            g.add_dev(self.synth.rows(r0, min(self.step, self.n - r0)))

    def fill(self, g, nlist, nprobe, reserve=False):
        """train shard g on the first 64 nlist rows (10 k-means iterations, at most 64 points per
        centroid), optionally reserve room for all n rows, add them, finalize and set nprobe; returns g"""
        g.set_param("kmeans_niter", 10)
        g.set_param("max_points_per_centroid", 64)
        g.train_dev(self.synth.rows(0, 64 * nlist))
        if reserve:
            g.reserve(self.n)
        self.add(g)
        g.finalize()
        g.nprobe = nprobe
        return g

    def exact(self, k):
        """the exact top-k ids of the queries, from a GPU flat (L2) index over the same rows that is
        built on the first call and freed before it returns"""
        if k not in self._exact:
            flat = engine.GpuIndex(engine.KIND_FLAT, self.d, engine.METRIC_L2)
            flat.reserve(self.n)
            self.add(flat)
            self._exact[k] = flat.search_dev(self.xq, k)[1].cpu().numpy()
            del flat
            torch.cuda.empty_cache()
        return self._exact[k]

    def recall(self, g, k):
        """recall@k of one search of the queries on shard g against the exact top-k"""
        exact = self.exact(k)
        I = g.search_dev(self.xq, k)[1].cpu().numpy()
        return float(np.mean([len(set(a) & set(b)) / k for a, b in zip(I, exact)]))


def mirror(o, g, nprobe):
    """oracle o holding shard g's state and probing nprobe lists; returns o"""
    o.set_state(g.get_state())
    o.nprobe = nprobe
    return o


def same_arrays(a, b):
    """whether two sequences of arrays, such as two (D, I) search results, are equal element for element"""
    return all(np.array_equal(x, y) for x, y in zip(a, b))


class SameLists:
    """Called on shards trained alike: whether each holds the centroids and list offsets of the first
    shard it was called on."""

    def __init__(self):
        self.first = None

    def __call__(self, g):
        lists = g.get_centroids(), g.get_array("list_off")
        if self.first is None:
            self.first = lists
        return same_arrays(lists, self.first)


def measure(g, xq, k, reps, refine=False):
    """One timed round of shard g on the batch xq: the batch ms (`timed`), then a profile window of reps
    searches for the list-scan ms per search (dfx_profile_*: the scan launch bracketed by CUDA events)
    and, with refine, the re-ranking ms per search (dfx_get_param "refine_ms").
    Returns (batch_ms, scan_ms, refine_ms or None, ndis)."""
    batch_ms = timed(lambda: g.search_dev(xq, k))
    g.profile(True)
    for _ in range(reps):
        g.search_dev(xq, k)
    torch.cuda.synchronize()
    refine_ms = g.get_param("refine_ms") / reps if refine else None
    scan_ms, _ = g.profile_read()
    g.profile(False)
    return batch_ms, scan_ms / reps, refine_ms, g.last_stats()["ndis"]


def time_rounds(cases, res, xq, k, rounds, reps):
    """Time resident shards in alternating rounds, so that the spread across rounds is visible.
    cases: (name, shard, k_factor, refine); a k_factor other than 0 is set on the shard before each of
    its rounds, so cases can share a shard; refine says whether the shard reports refine_ms.
    res[name] collects each round's ms in *_ms_rounds lists and the shard's ndis, then gains the
    medians, the [min, max] of the scan (and refine) ms and the qps."""
    for name, _, _, _ in cases:
        for key in ("batch_ms_rounds", "scan_kernel_ms_rounds", "refine_ms_rounds"):
            res[name].setdefault(key, [])
    for _ in range(rounds):
        for name, g, k_factor, refine in cases:
            if k_factor:
                g.set_param("k_factor", k_factor)
            batch_ms, scan_ms, refine_ms, ndis = measure(g, xq, k, reps, refine)
            r = res[name]
            r["batch_ms_rounds"].append(batch_ms)
            r["scan_kernel_ms_rounds"].append(scan_ms)
            if refine:
                r["refine_ms_rounds"].append(refine_ms)
            r["ndis"] = ndis
    for name, _, _, refine in cases:
        r = res[name]
        r.update({
            "batch_ms": float(np.median(r["batch_ms_rounds"])),
            "scan_kernel_ms": float(np.median(r["scan_kernel_ms_rounds"])),
            "scan_kernel_ms_min_max": [min(r["scan_kernel_ms_rounds"]), max(r["scan_kernel_ms_rounds"])],
            "qps": len(xq) / float(np.median(r["batch_ms_rounds"])) * 1e3,
        })
        if refine:
            r["refine_ms"] = float(np.median(r["refine_ms_rounds"]))
            r["refine_ms_min_max"] = [min(r["refine_ms_rounds"]), max(r["refine_ms_rounds"])]
        else:
            del r["refine_ms_rounds"]
