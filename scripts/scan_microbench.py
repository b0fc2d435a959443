#!/usr/bin/env python
"""One shard of the bench workload (62.5 M vectors of the 500 M, nlist 65 536), batch 4096, nprobe 8:
per-launch time of the fused table-build + scan kernel and of the whole shard search, for the
kernel knobs currently in the environment (DFX_IL2_PREFETCH ...), then a per-kernel breakdown of
one shard search from torch.profiler (MB_PROFILE=0 skips it).  ~60 s per run.
    python scripts/scan_microbench.py [label]"""
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402
from distributed_faiss_b200 import engine  # noqa: E402


class A:
    nlist = 0
    kmeans_niter = 10
    train_pts = 64


# the kernels of one IVF-PQ shard search, in launch order
BREAKDOWN_KERNELS = ("f16_rows_kernel", "tc_coarse_kernel", "decide_rows_kernel", "tc_exact_rows_kernel",
                     "scan_pq_il2_kernel")
TC_PEAK_TFLOPS = 989.0  # H100 SXM data sheet, dense fp16 with fp32 accumulation


def card_info():
    """name, power limit and maximum SM clock of the card (a read-only query)."""
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader",
                            "-i", str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30)
        return r.stdout.strip()
    except (OSError, subprocess.SubprocessError) as e:
        return f"nvidia-smi failed: {e}"


def kernel_breakdown(idx, batch, k, iters=20):
    """Per-kernel device time of `iters` shard searches of `batch` (torch.profiler, CUDA activities),
    against the search's own time measured with the profiler off, and the SM clock sampled while
    the searches ran.  K1 (tc_coarse_kernel) also gets its algorithmic rate 2 nq_pad nl_pad d and
    its MMA rate (x3 for PRECISE: three products per k-step)."""
    from torch.profiler import ProfilerActivity, profile

    for _ in range(3):
        idx.search_dev(batch, k)
    torch.cuda.synchronize()
    clocks = bench.ClockSampler(torch.cuda.current_device())
    clocks.start()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        idx.search_dev(batch, k)
    e1.record()
    torch.cuda.synchronize()
    search_us = e0.elapsed_time(e1) * 1e3 / iters
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(iters):
            idx.search_dev(batch, k)
        torch.cuda.synchronize()
    clk = clocks.stop()
    per = {}
    for ev in prof.key_averages():
        name = next((kn for kn in BREAKDOWN_KERNELS if kn in ev.key), None)
        if name is None or ev.device_time_total <= 0:
            continue
        p = per.setdefault(name, {"launches": 0, "total_us": 0.0})
        p["launches"] += ev.count
        p["total_us"] += ev.device_time_total
    out = {"search_us": search_us, "sm_clock": clk, "kernels": {}}
    for name in BREAKDOWN_KERNELS:
        p = per.get(name, {"launches": 0, "total_us": 0.0})
        launches_per_search = p["launches"] / iters
        us_search = p["total_us"] / iters
        out["kernels"][name] = {"us_per_launch": p["total_us"] / p["launches"] if p["launches"] else 0.0,
                                "launches_per_search": launches_per_search, "us_per_search": us_search,
                                "share_of_search": us_search / search_us}
    k1 = out["kernels"]["tc_coarse_kernel"]
    if k1["launches_per_search"]:
        nq_pad = -(-batch.shape[0] // 128) * 128
        nl_pad = -(-idx.nlist // 128) * 128
        flop = 2.0 * nq_pad * nl_pad * batch.shape[1] * k1["launches_per_search"]
        products = 1 if idx.get_param("tc_fast") else 3
        t = k1["us_per_search"] * 1e-6
        k1["algorithmic_tflops"] = flop / t / 1e12
        k1["mma_tflops"] = products * flop / t / 1e12
        k1["mma_frac_of_989"] = k1["mma_tflops"] / TC_PEAK_TFLOPS
    return out


def screen_tol(d, fast, qn2, cmax2, qn2c=None, cmax2c=None):
    """dfx_tc.cu's screening tolerance of a row: raw (qn2c None) as before centring, i.e.
    4.2 err |q| max|c| + 1e-5 (max|c|^2 + 2 |q| max|c|), or centred on the centroid mean m."""
    err = (2.0 ** -10 + 2.0 ** -22 + d * 2.0 ** -24) if fast else (3 * 2.0 ** -22 + 3 * d * 2.0 ** -24)
    s = (qn2 * cmax2).sqrt()
    if qn2c is None:
        return 4.2 * err * s + 1e-5 * (cmax2 + 2 * s)
    sc = (qn2c * cmax2c).sqrt()
    return (4.2 * (err + 2.0 ** -23) * sc + 2.1 * (2.0 ** -18 + 2.0 ** -23) * (cmax2c + 2 * sc)
            + 2.1 * (2.0 ** -17 + 2.0 ** -22 + d * 2.0 ** -24) * (cmax2 + 2 * s))


def fast_overflow_rates(synth, nvec, cent, cn, nprobe, nrows=32768, margins=(8, 16, 24)):
    """Share of `nrows` bench queries whose decide stage would overflow under FAST's tolerance:
    the G-th smallest group minimum (exact fp32 ranking values |c|^2 - 2 q.c, groups of 32
    centroids) within the tolerance of the nprobe-th one, G = nprobe + margin.  Raw tolerance
    and tolerance centred on the centroid mean."""
    g = torch.Generator(device="cpu").manual_seed(1237)
    rows = torch.randint(0, nvec, (nrows,), generator=g, dtype=torch.int64).cuda()
    xq = synth.rows(0, nrows, rows_t=rows, noise_stream=7)
    d, nl = cent.shape[1], cent.shape[0]
    m = cent.double().mean(0).float()
    cmax2, cmax2c = float(cn.max()), float(((cent - m) ** 2).sum(1).max())
    Gmax = nprobe + max(margins)
    cases = {"raw_G+8": [], **{f"centred_G+{mg}": [] for mg in margins}}
    tol_med = {"raw": [], "centred": []}
    for r0 in range(0, nrows, 2048):
        q = xq[r0:r0 + 2048]
        gm = (cn[None, :] - 2.0 * q @ cent.t())[:, :nl // 32 * 32].view(q.shape[0], -1, 32).amin(2)
        top = torch.topk(gm, Gmax, dim=1, largest=False, sorted=True).values.double()
        t = top[:, nprobe - 1]
        qn2, qn2c = (q.double() ** 2).sum(1), ((q - m).double() ** 2).sum(1)
        tr = screen_tol(d, True, qn2, cmax2)
        tc = screen_tol(d, True, qn2, cmax2, qn2c, cmax2c)
        tol_med["raw"].append(tr)
        tol_med["centred"].append(tc)
        cases["raw_G+8"].append(top[:, nprobe + 8 - 1] <= t + tr)
        for mg in margins:
            cases[f"centred_G+{mg}"].append(top[:, nprobe + mg - 1] <= t + tc)
    out = {"rows": nrows, "nprobe": nprobe, "cmax2": cmax2, "cmax2_centred": cmax2c,
           "qnorm_centred_mean": float(((xq - m) ** 2).sum(1).sqrt().mean())}
    for k, v in cases.items():
        v = torch.cat(v)
        out[k] = {"overflow_rows": int(v.sum()), "share": float(v.double().mean())}
    for k, v in tol_med.items():
        out[f"tol_median_{k}"] = float(torch.cat(v).median())
    return out


def main():
    label = sys.argv[1] if len(sys.argv) > 1 else "default"
    nvec = int(os.environ.get("MB_NVEC", 500_000_000))
    G = nvec // 10
    synth = engine.Synth(1234, bench.D, 16, 1, 1.0, 0.02, ngroups=G, eps=0.01, delta=0.1)
    idx, tab, info = bench.build_shard(engine, synth, nvec, 0, A, torch, None)
    g = torch.Generator(device="cpu").manual_seed(1236)
    q_rows = torch.randint(0, nvec, (12288,), generator=g, dtype=torch.int64).cuda()
    xq = synth.rows(0, 12288, rows_t=q_rows, noise_stream=7)
    idx.nprobe = int(os.environ.get("MB_NPROBE", 8))
    out = {"label": label, "info": info}
    # MB_VARIANTS="threads:prefetch,..." e.g. "256:4,256:0,512:4" (dfx_set_param il2_threads / il2_prefetch)
    variants = [tuple(int(x) for x in v.split(":")) for v in os.environ.get("MB_VARIANTS", "0:-1").split(",")]
    ref = None
    B = 4096
    batches = [xq[i * B:(i + 1) * B].contiguous() for i in range(12288 // B)]
    reps = int(os.environ.get("MB_REPS", 3))
    acc = {}
    # round robin over the variants, `reps` times: clocks drift under sustained load, so a variant
    # is only comparable with its neighbours in time; the median over the rounds is reported
    for rep in range(reps):
        for (thr, pf) in variants:
            idx.set_param("il2_threads", thr)
            idx.set_param("il2_prefetch", pf)
            for b in batches:
                Dv, Iv = idx.search_dev(b, 10)
            torch.cuda.synchronize()
            if ref is None:
                ref = (Dv.clone(), Iv.clone())
            same = bool(torch.equal(Dv, ref[0]) and torch.equal(Iv, ref[1]))
            ndis = idx.last_stats()["ndis"]
            idx.profile(True)
            idx.profile_read(True)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            last = rep == reps - 1 and (thr, pf) == variants[-1]
            if last:
                torch.cuda.profiler.start()   # ncu --profile-from-start off: the launch list of one variant
            e0.record()
            n = 12
            for i in range(n):
                idx.search_dev(batches[i % len(batches)], 10)
            e1.record()
            torch.cuda.synchronize()
            if last:
                torch.cuda.profiler.stop()
            ms, nl = idx.profile_read(True)
            idx.profile(False)
            a = acc.setdefault(f"t{thr}_pf{pf}", {"scan_ms": [], "search_ms": [], "same": True, "ndis": ndis})
            a["scan_ms"].append(ms / nl)
            a["search_ms"].append(e0.elapsed_time(e1) / n)
            a["same"] = a["same"] and same
    for k, a in acc.items():
        sm = float(np.median(a["scan_ms"]))
        out[k] = {"same_as_first_variant": a["same"], "scan_ms_per_launch": sm, "scan_ms_all": a["scan_ms"],
                  "search_ms": float(np.median(a["search_ms"])), "algorithmic_GBps": a["ndis"] * 32 / sm / 1e6,
                  "frac_of_3350": a["ndis"] * 32 / sm / 1e6 / 3350.0}
    # the distribution the screening tolerance is up against: gaps between the 8th, 9th and 16th
    # smallest ranking values |c|^2 - 2 q.c of a query sample (exact fp32, torch)
    cent = torch.from_numpy(idx.get_array("centroids").reshape(-1, bench.D)).cuda()
    cn = (cent * cent).sum(1)
    qs = batches[0][:512]
    V = cn[None, :] - 2.0 * qs @ cent.t()
    Vs = torch.sort(V, dim=1).values[:, :32]
    qn = (qs * qs).sum(1).sqrt()
    def qtl(t):
        return [float(torch.quantile(t, q)) for q in (0.01, 0.1, 0.5, 0.9)]
    out["gap_stats"] = {"cmax2": float(cn.max()), "cmean2": float(cn.mean()), "qnorm_mean": float(qn.mean()),
                        "tc_cmax2": idx.get_param("tc_cmax2"),
                        "gap_8_to_9": qtl(Vs[:, 8] - Vs[:, 7]), "gap_8_to_16": qtl(Vs[:, 15] - Vs[:, 7]),
                        "gap_8_to_24": qtl(Vs[:, 23] - Vs[:, 7]), "v8": qtl(Vs[:, 7])}
    del V, Vs
    out["fast_overflow"] = fast_overflow_rates(synth, nvec, cent, cn, idx.nprobe)
    # coarse-quantizer screening precision: AUTO state after the runs above, then the fixed modes
    stat_names = ("tc_fast", "tc_stat_rows", "tc_stat_overflow", "tc_stat_fast_would")
    out["auto_state"] = {k: idx.get_param(k) for k in stat_names}
    for mode, name in ((2, "precise"), (1, "fast"), (0, "auto")):
        idx.set_param("tc_screen_mode", mode)
        for b in batches:
            idx.search_dev(b, 10)
        torch.cuda.synchronize()
        idx.profile(True)
        idx.profile_read(True)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for i in range(12):
            Dm, Im = idx.search_dev(batches[i % len(batches)], 10)
        e1.record()
        torch.cuda.synchronize()
        ms, nl = idx.profile_read(True)
        idx.profile(False)
        Dm, Im = idx.search_dev(batches[-1], 10)
        out["screen_" + name] = {"search_ms": e0.elapsed_time(e1) / 12, "scan_ms": ms / nl,
                                 "coarse_ms": e0.elapsed_time(e1) / 12 - ms / nl,
                                 "same": bool(torch.equal(Dm, ref[0]) and torch.equal(Im, ref[1])),
                                 **{k: idx.get_param(k) for k in stat_names}}
        if os.environ.get("MB_PROFILE", "1") != "0" and mode != 0:
            out["breakdown_" + name] = kernel_breakdown(idx, batches[0], 10)
    if os.environ.get("MB_PROFILE", "1") != "0":  # AUTO, as left by the loop above
        out["card"] = card_info()
        out["breakdown"] = kernel_breakdown(idx, batches[0], 10)
        out["breakdown"]["auto_state"] = {k: idx.get_param(k) for k in stat_names}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
