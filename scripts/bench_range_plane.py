#!/usr/bin/env python
"""IndexClient.range_search over the search plane against the sockets (one H100, four IndexServers).

Four IndexServers in this process on cuda:0 under one SearchPlane, as the GPU tests set them up, each
holding one shard of the bench generator (kind_bench.Dataset "bench", near-duplicate groups of 10) with
integer metadata:
  ivf_pq    8-bit IVF-PQ, d = 128, 2 M vectors per server, nlist 2048, M = 32, nprobe 32
  sqfp16    SQfp16 flat (L2), d = 768, 250 000 vectors per server
1 000 queries.  Radii (one per call; per-query radii are not served): the median over the queries of the
10th and of the 100th neighbour's distance of the merged k-NN search, and a radius that returns about
10 000 hits per query (the median over 20 queries of their 10 000th distance).
Per configuration, before any time is taken, the plane's and the sockets' (lims, scores, metadata) must
be equal bit for bit.  Then, in alternating rounds, the wall time of one `range_search` call over the
1 000 host queries (host arrays out, so every call ends synchronised) over the plane and over the sockets:
median and [min, max].  In a separate run, torch.profiler gives the device time of the merge kernel
(range_merge_kernel and range_merge_lims_kernel) of one plane call, reported as a share of the plane's
median call time.  The card name and its power limit are recorded with the numbers."""
import json
import os
import socket
import sys
import tempfile
import threading
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))
import kind_bench as kb  # noqa: E402
from distributed_faiss_b200 import engine, spmd  # noqa: E402
from distributed_faiss_b200.client import IndexClient  # noqa: E402
from distributed_faiss_b200.index_cfg import IndexCfg  # noqa: E402
from distributed_faiss_b200.server import IndexServer  # noqa: E402

N_SERVERS, NQ, ROUNDS = 4, 1000, 3


def cluster(store):
    socks = [socket.socket() for _ in range(N_SERVERS)]
    for s in socks:
        s.bind(("127.0.0.1", 0))
    ports = [s.getsockname()[1] for s in socks]
    for s in socks:
        s.close()
    servers = []
    for rank, port in enumerate(ports):
        srv = IndexServer(rank, store, device=0)
        threading.Thread(target=srv.start_blocking, args=(port,), daemon=True).start()
        servers.append(srv)
    for p in ports:
        while True:
            try:
                socket.create_connection(("127.0.0.1", p), timeout=1.0).close()
                break
            except OSError:
                time.sleep(0.05)
    plane = spmd.SearchPlane(servers)
    disc = os.path.join(store, "servers.txt")
    with open(disc, "w") as fh:
        fh.write(f"{N_SERVERS}\n" + "".join(f"localhost,{p}\n" for p in ports))
    client = IndexClient(disc)
    assert client.plane is plane
    return servers, plane, client


def build(servers, name, kind, d, n, cfg, **kw):
    ds = kb.Dataset(d, N_SERVERS * n, NQ, step=250_000)
    for j, srv in enumerate(servers):
        if kind == engine.KIND_IVF_PQ:
            g = engine.GpuIndex(kind, d, engine.METRIC_L2, nlist=kw["nlist"], pq_m=kw["M"])
            g.set_param("kmeans_niter", 10)
            g.set_param("max_points_per_centroid", 64)
            g.train_dev(ds.synth.rows(0, 64 * kw["nlist"]))
        else:
            g = engine.GpuIndex(kind, d, engine.METRIC_L2)
        g.reserve(n)
        for r0 in range(0, n, ds.step):
            g.add_dev(ds.synth.rows(j * n + r0, min(ds.step, n - r0)))
        g.finalize()
        if kind == engine.KIND_IVF_PQ:
            g.nprobe = kw["nprobe"]
        srv.adopt_index(name, cfg, g, torch.arange(j * n, (j + 1) * n, dtype=torch.int64, device="cuda:0"))
    return ds.xq.cpu().numpy()


def both(client, plane, fn):
    client.plane = plane
    a = fn()
    client.detach_plane()
    b = fn()
    client.plane = plane
    return a, b


def wall(fn):
    t0 = time.perf_counter()
    fn()
    return 1e3 * (time.perf_counter() - t0)


def merge_ms(client, xq, r, name):
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        client.range_search(xq, r, name)
        torch.cuda.synchronize()
    us = sum(e.device_time_total for e in prof.key_averages() if "range_merge" in e.key)
    return us / 1e3


def main():
    out = {"card": kb.card(), "setup": {"servers": N_SERVERS, "nq": NQ, "rounds": ROUNDS,
                                        "dataset": "bench (near-duplicate groups of 10)"}}
    store = tempfile.TemporaryDirectory()
    servers, plane, client = cluster(store.name)
    configs = [("ivf_pq", engine.KIND_IVF_PQ, 128, 2_000_000,
                IndexCfg(index_builder_type="knnlm", dim=128, metric="l2", centroids=2048, code_size=32),
                dict(nlist=2048, M=32, nprobe=32)),
               ("sqfp16", engine.KIND_FLAT_SQ16, 768, 250_000, IndexCfg(faiss_factory="SQfp16", dim=768, metric="l2"),
                {})]
    try:
        for name, kind, d, n, cfg, kw in configs:
            xq = build(servers, name, kind, d, n, cfg, **kw)
            client.cfg = cfg
            D, _ = client.search(xq, 100, name)
            full = client.range_search(xq[:20], np.inf, name)
            r_1e4 = float(np.median([np.sort(full[1][full[0][q]:full[0][q + 1]])[9999] for q in range(20)]))
            radii = {"r10": float(np.median(D[:, 9])), "r100": float(np.median(D[:, 99])), "r1e4": r_1e4}
            res = {}
            for rname, r in radii.items():
                a, b = both(client, plane, lambda: client.range_search(xq, r, name))
                same = (np.array_equal(a[0], b[0]) and np.array_equal(a[1].view(np.int32), b[1].view(np.int32))
                        and list(a[2]) == list(b[2]))
                if not same:
                    raise SystemExit(f"{name} {rname}: the plane and the sockets differ")
                t = {"plane": [], "sockets": []}
                for _ in range(ROUNDS):
                    tp, ts = both(client, plane, lambda: wall(lambda: client.range_search(xq, r, name)))
                    t["plane"].append(tp)
                    t["sockets"].append(ts)
                res[rname] = {"radius": r, "hits_per_query": float(a[0][-1]) / NQ,
                              "max_hits": int(np.diff(a[0]).max())}
                for path, v in t.items():
                    res[rname][f"{path}_ms"] = {"median": float(np.median(v)), "min": float(min(v)),
                                                "max": float(max(v))}
            for rname, r in radii.items():   # the profiled runs, after every timed round
                m = merge_ms(client, xq, r, name)
                res[rname]["merge_kernel_ms"] = m
                res[rname]["merge_share_of_plane"] = m / res[rname]["plane_ms"]["median"]
            out[name] = res
            for srv in servers:
                srv.indexes.pop(name, None)
            torch.cuda.empty_cache()
    finally:
        client.close()
        plane.stop()
        for s in servers:
            s.stop()
    print(json.dumps(out, indent=1))


if __name__ == "__main__":
    main()
