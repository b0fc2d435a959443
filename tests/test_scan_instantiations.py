"""Every compiled instantiation of the IVF list scans against the oracle, bit for bit.

Each list-scan family is one template compiled once per shape (code width, CTA shape, rows in flight,
k > 1024), and each instantiation is its own machine code that a shard can select.  SCANS maps every
instantiation, named as `nm -C` prints it, to a shard and searches that select it:

  * the shard is built by the oracle (train_niter = 2) and imported, so the case is the same small
    shard on the GPU and on the emulator.  Its centroids are orthogonal and well separated, so the
    list lengths are chosen: an empty list, 1, 31 and 33 rows, THREADS - 1 and THREADS + 1 rows, and
    one list that fills k = 1024 at nprobe 1.  One list holds exact duplicate rows, and the ids are
    renumbered to descend inside every list, so that ties follow the id and not the row position.
  * the queries are clustered queries, the duplicated row itself, and one query equidistant from
    every centroid (it probes the empty list at nprobe 1).
  * the searches run nprobe in {1, 3, nlist} and k values on both sides of the queue sizes, within the
    range of k that selects the case's instantiation.

CPU: the keys of SCANS are exactly the instantiations the library compiles (the emulator build, and
libdfx.so when it is current), and this file's `gpu` tests run against the emulated library, where
every search also asserts that it launched the case's instantiation and no other list scan.  The
planner's only device-dependent input is the shared memory one block may opt in to: the GPU run
asserts the H100's value, the one the emulator reports, so the routing proven there holds on the H100.
"""
import ctypes as C
import os
import platform
import re
import shutil
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
IP, L2 = 0, 1
FMAX = np.finfo(np.float32).max
EMU = bool(os.environ.get("DFX_EMU_LIB"))
SMEM_OPTIN = 232448  # bytes one block may opt in to on sm_90 (227 KB)
SCAN_NAME = re.compile(r"\bscan_\w+_kernel<[^>]*>")


def _sz(full, emu):
    return emu if EMU else full


# ------------------------------------------------------------------ the table
def _case(kind, metric, d, ks, M=0, nbits=8, threads=128, **params):
    """kind and metric (the coarse quantizer's; IVF-Flat scans by it too), the shard's shape, the k
    values searched, the CTA size of the scan (the list lengths straddle it) and engine parameters
    (interleaved, rows_inflight, il2_threads)"""
    assert ks, "a case searches at least one k"
    return dict(kind=kind, metric=metric, d=d, M=M, nbits=nbits, threads=threads, ks=tuple(ks), params=params)


KS = (1, 32, 33, 1024)           # 128-thread queues: k = 1, one warp's 32, past it, the largest
KS_MAT = (1025, 2049, 4096)      # k > 1024: every composite to a candidate row


def _wide_threads(M, k):
    """the CTA shape the planner gives the wide scan: the widest whose table and queues fit"""
    cap = 2 * max(32, 1 << (k - 1).bit_length())
    return next((t for t in (512, 256, 128) if M * 256 * 4 + (t // 32) * cap * 8 <= SMEM_OPTIN), 0)


def _wide_ks(M, threads):
    return [k for k in (1, 32, 33, 256, 257, 512, 513, 1024) if _wide_threads(M, k) == threads]


SCANS = {}
# scan_rows_kernel<MODE, U, MAT>: MODE 0 / 1 IVF-Flat by IP / L2, 2 IVF-SQ fp16, 3 IVF-SQ8; U = 8 rows in
# flight per warp for rows of up to 1 KB, else 4.  d is not a multiple of 32 (100, 36) or of 128 (1028, 516).
for mode, (kind, metric) in enumerate([("ivf_flat", IP), ("ivf_flat", L2), ("ivf_sq", L2), ("ivf_sq8", L2)]):
    SCANS[f"scan_rows_kernel<{mode}, 8, false>"] = _case(kind, metric, 100, KS)
    SCANS[f"scan_rows_kernel<{mode}, 8, true>"] = _case(kind, metric, 36, KS_MAT)
    SCANS[f"scan_rows_kernel<{mode}, 4, false>"] = _case(kind, metric, 1028, KS)
    # 516 B of SQ8 codes would take 8 rows in flight: the knob asks for 4
    SCANS[f"scan_rows_kernel<{mode}, 4, true>"] = _case(kind, metric, 516, KS_MAT,
                                                       **({"rows_inflight": 4} if mode == 3 else {}))
# scan_pq_kernel<MT, MAT>: 8-bit codes, row-major, M <= 64; MT = 0 for any M but 8, 16, 32, 64
for mt, (M, d), (Mm, dm) in [(8, (8, 40), (8, 24)), (16, (16, 48), (16, 16)), (32, (32, 64), (32, 96)),
                             (64, (64, 128), (64, 64)), (0, (60, 120), (4, 36))]:
    il = {"interleaved": 0} if mt == 32 else {}  # M = 32 is interleaved by default (scan_pq_il2_kernel)
    SCANS[f"scan_pq_kernel<{mt}, false>"] = _case("ivf_pq", L2, d, KS, M=M, **il)
    SCANS[f"scan_pq_kernel<{mt}, true>"] = _case("ivf_pq", L2, dm, KS_MAT, M=Mm, **il)
# scan_pq_wide_kernel<MT, THREADS, MAT>: 64 < M <= 128; THREADS by k (_wide_threads); MT = 0 for M but 96, 128
for mt, threads, M, d in [(128, 512, 128, 256), (128, 256, 128, 128), (128, 128, 128, 384), (96, 512, 96, 288),
                          (96, 256, 96, 96), (0, 512, 68, 204), (0, 256, 72, 360), (0, 128, 100, 200)]:
    SCANS[f"scan_pq_wide_kernel<{mt}, {threads}, false>"] = _case("ivf_pq", L2, d, _wide_ks(M, threads), M=M,
                                                                  threads=threads)
for mt, M, d in [(128, 128, 128), (96, 96, 192), (0, 116, 232)]:
    SCANS[f"scan_pq_wide_kernel<{mt}, 512, true>"] = _case("ivf_pq", L2, d, KS_MAT, M=M, threads=512)
# scan_pq4_kernel<M, MAT> (4-bit IVF-PQ) and scan_pq_fs_kernel<M, MAT> (FastScan): M = 8, 16, ..., 128
for i, M in enumerate(range(8, 129, 8)):
    for kind, nbits, name in [("ivf_pq", 4, "scan_pq4_kernel"), ("ivf_pq_fs", 4, "scan_pq_fs_kernel")]:
        SCANS[f"{name}<{M}, false>"] = _case(kind, L2, M * (2, 3, 1)[i % 3], KS, M=M, nbits=nbits)
        SCANS[f"{name}<{M}, true>"] = _case(kind, L2, M * (1, 2, 3)[i % 3], KS_MAT, M=M, nbits=nbits)
# scan_pq_il2_kernel<REG, THREADS, MINB, MAT>: 8-bit M = 32, interleaved; REG for k <= 32; 512 threads
# (il2_threads) only while 16 queues fit, k <= 512
SCANS["scan_pq_il2_kernel<true, 256, 3, false>"] = _case("ivf_pq", L2, 64, (1, 32), M=32, threads=256)
SCANS["scan_pq_il2_kernel<true, 512, 2, false>"] = _case("ivf_pq", L2, 96, (1, 32), M=32, threads=512,
                                                         il2_threads=512)
SCANS["scan_pq_il2_kernel<false, 256, 3, false>"] = _case("ivf_pq", L2, 160, (33, 513, 1024), M=32, threads=256)
SCANS["scan_pq_il2_kernel<false, 512, 2, false>"] = _case("ivf_pq", L2, 32, (33, 512), M=32, threads=512,
                                                          il2_threads=512)
SCANS["scan_pq_il2_kernel<false, 256, 3, true>"] = _case("ivf_pq", L2, 128, KS_MAT, M=32, threads=256)


# ------------------------------------------------------------------ coverage (CPU)
def _emu_build():
    if shutil.which("g++") is None or platform.machine() != "x86_64":
        pytest.skip("the emulator needs g++ on x86-64")
    sys.path.insert(0, os.path.join(ROOT, "tests", "emu"))
    try:
        import build_emu_lib
    finally:
        sys.path.pop(0)
    return build_emu_lib.build()


def _scan_symbols(path, dynamic):
    out = subprocess.run(["nm", "-C"] + (["-D"] if dynamic else []) + [path], capture_output=True, text=True,
                         check=True).stdout
    return set(SCAN_NAME.findall(out))


def test_scans_table_is_every_compiled_instantiation():
    """a new instantiation without a case fails, and so does a case for a kernel that does not exist"""
    if shutil.which("nm") is None:
        pytest.skip("nm is not available")
    emu = _scan_symbols(_emu_build(), dynamic=True)
    assert emu == set(SCANS), (f"compiled without a case: {sorted(emu - set(SCANS))}; "
                               f"cases without a kernel: {sorted(set(SCANS) - emu)}")
    from distributed_faiss_b200 import build

    if os.path.exists(build.LIB) and build.is_current():
        assert _scan_symbols(build.LIB, dynamic=False) == emu


def test_scan_instantiations_on_the_emulated_library():
    env = dict(os.environ, DFX_EMU_LIB=_emu_build())
    run = subprocess.run([sys.executable, "-m", "pytest", "-m", "gpu", "-q", "-x", "-p", "no:cacheprovider",
                          os.path.abspath(__file__)], cwd=ROOT, env=env, capture_output=True, text=True, timeout=3000)
    tail = (run.stdout + run.stderr)[-3000:]
    assert run.returncode == 0, tail
    assert f"{len(SCANS)} passed" in run.stdout, tail


# ------------------------------------------------------------------ the sweep
def _launched_scans():
    """the list scans launched since the last call (emulated library only)"""
    from distributed_faiss_b200 import engine

    f = engine.lib().dfx_emu_launch_log
    f.restype, f.argtypes = C.c_int64, [C.c_char_p, C.c_int64]
    while True:
        n = f(None, 0)
        buf = C.create_string_buffer(n)
        if f(buf, n) <= n:
            return SCAN_NAME.findall(buf.value.decode())


def _shard(c, rs):
    """(GpuIndex, oracle, queries) of case c: the list lengths of the module docstring"""
    from distributed_faiss_b200 import engine as E
    from tests.oracle_pq_fs import make_index

    d, T = c["d"], c["threads"]
    sizes = [0, 1, 31, 33, T - 1, T + 1, _sz(1100, 1030)]
    nlist = len(sizes)
    cent = np.zeros((nlist, d), dtype=np.float32)
    cent[np.arange(nlist), np.arange(nlist)] = 10.0           # orthogonal, |c| equal: both metrics separate them
    x = np.concatenate([cent[l] + 0.5 * rs.randn(s, d).astype(np.float32) for l, s in enumerate(sizes)])
    x = x.astype(np.float32)
    # exact duplicates in the long list, side by side and spread over it: the later copies reach a
    # warp after its queue was cut at their value, and they hold the smaller ids
    dup = len(x) - sizes[-1]
    x[dup + np.r_[1:5, 97:sizes[-1]:97]] = x[dup]
    o = make_index(c["kind"], d, metric=c["metric"], nlist=nlist, M=c["M"], nbits=c["nbits"])
    o.train_niter = 2
    o.train(x)
    o.centroids = cent.copy()
    o.add(x)
    assert np.diff(o.list_off).tolist() == sizes
    st = o.get_state()
    ids = st["ids"].copy()
    for b, e in zip(st["list_off"][:-1], st["list_off"][1:]):
        ids[b:e] = ids[b:e][::-1]                              # descending inside every list
    st["ids"] = ids
    o.set_state(st)
    kinds = {"ivf_flat": E.KIND_IVF_FLAT, "ivf_sq": E.KIND_IVF_SQ16, "ivf_sq8": E.KIND_IVF_SQ8,
             "ivf_pq": E.KIND_IVF_PQ, "ivf_pq_fs": E.KIND_IVF_PQ_FS}
    g = E.GpuIndex(kinds[c["kind"]], d, c["metric"], nlist=nlist, pq_m=c["M"], pq_nbits=c["nbits"])
    for name, value in c["params"].items():
        g.set_param(name, value)
    g.set_state(st)
    far = np.zeros((1, d), dtype=np.float32)
    far[0, nlist] = -30.0                                      # equidistant from every centroid: probes list 0
    xq = np.concatenate([cent[[6, 5, 2]] + 0.5 * rs.randn(3, d).astype(np.float32), x[dup:dup + 1], far])
    return g, o, xq.astype(np.float32)


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(SCANS), ids=lambda s: re.sub(r"[<>, ]+", "-", s).strip("-"))
def test_scan_instantiation_matches_oracle(name):
    """distances, ids and ndis bit for bit; on the emulator each search launches `name` and no other
    list scan"""
    if not EMU:
        import torch

        assert torch.cuda.get_device_properties(0).shared_memory_per_block_optin == SMEM_OPTIN
    c = SCANS[name]
    g, o, xq = _shard(c, np.random.RandomState(sorted(SCANS).index(name)))
    pad = -FMAX if (c["kind"] == "ivf_flat" and c["metric"] == IP) else FMAX
    if EMU:
        _launched_scans()
    for nprobe in (1, 3, g.nlist):
        g.nprobe = o.nprobe = nprobe
        for k in c["ks"]:
            what = f"{name} nprobe={nprobe} k={k}"
            Dg, Ig = g.search(xq, k)
            if EMU:
                assert _launched_scans() == [name], what
            Do, Io = o.search(xq, k)
            if not (np.array_equal(Ig, Io) and np.array_equal(Dg, Do)):
                bad = np.argwhere((Ig != Io) | (Dg != Do))
                q, j = bad[0]
                raise AssertionError(f"{what}: {len(bad)} mismatching slots of {Ig.size}; first at q={q} j={j}: "
                                     f"gpu=({Dg[q, j]!r},{Ig[q, j]}) oracle=({Do[q, j]!r},{Io[q, j]})")
            assert g.last_stats()["ndis"] == o.last_ndis, what
            if nprobe == 1:
                assert (Ig[-1] == -1).all() and (Ig[-1] == Io[-1]).all(), what     # the empty list
                assert (Dg[Ig == -1] == pad).all(), what
