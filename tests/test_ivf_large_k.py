"""IVF search with 1024 < k <= 4096: the list scans write every probed vector's composite to its
slot of the query's candidate row (MAT = true) and one k-selection per query picks the result
(dfx_search.cu, cand_offsets_kernel / select_cand_kernel).

Every case is compared bit for bit with the C oracle: distances, ids, the (value asc, id asc) order,
(+-FLT_MAX, -1) padding, and ndis.

CPU: the client's limit, and this file's `gpu` tests run against the emulated library.
GPU: every list scan and code layout, both coarse paths, query chunks, the per-query budget, and
two knnlm servers through the client over sockets and over the search plane."""
import os
import platform
import shutil
import subprocess
import sys

import numpy as np
import pytest

from tests.conftest import clustered
from tests import oracle_sq8 as S

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
IP, L2 = 0, 1
FMAX = np.finfo(np.float32).max
EMU = bool(os.environ.get("DFX_EMU_LIB"))
KS = [1025, 2048, 2049, 4096]
CAND_BUDGET = 128 << 20          # bytes of candidate rows one IVF query chunk may hold

# name: (kind, metric, d, M, nbits, interleaved)
KINDS = {
    "flat_ip": ("ivf_flat", IP, 64, 0, 8, None),
    "flat_l2": ("ivf_flat", L2, 64, 0, 8, None),
    "sq16": ("ivf_sq", L2, 64, 0, 8, None),
    "sq8": ("ivf_sq8", L2, 64, 0, 8, None),
    "pq32_interleaved": ("ivf_pq", L2, 128, 32, 8, 1),
    "pq32_row_major": ("ivf_pq", L2, 128, 32, 8, 0),
    "pq8": ("ivf_pq", L2, 64, 8, 8, None),
    "pq16": ("ivf_pq", L2, 64, 16, 8, None),
    "pq24": ("ivf_pq", L2, 96, 24, 8, None),
    "pq64": ("ivf_pq", L2, 128, 64, 8, None),
    "pq96": ("ivf_pq", L2, 384, 96, 8, None),
    "pq128": ("ivf_pq", L2, 512, 128, 8, None),
    "pq4_16": ("ivf_pq", L2, 64, 16, 4, None),
    "pq4_32": ("ivf_pq", L2, 128, 32, 4, None),
}


def _sz(full, emu):
    return emu if EMU else full


def _engine():
    from distributed_faiss_b200 import engine

    return engine


def _assert_same(Dg, Ig, Do, Io, what):
    if not (np.array_equal(Ig, Io) and np.array_equal(Dg, Do)):
        bad = np.argwhere((Ig != Io) | (Dg != Do))
        q, j = bad[0]
        raise AssertionError(f"{what}: {len(bad)} mismatching slots of {Ig.size}; first at q={q} j={j}: "
                             f"gpu=({Dg[q, j]!r},{Ig[q, j]}) oracle=({Do[q, j]!r},{Io[q, j]})")


def _pad_value(kind, metric):
    """the padding distance: the scan metric is IP only for IVF-Flat IP"""
    return -FMAX if (kind == "ivf_flat" and metric == IP) else FMAX


def _pair(name, nlist, n, rs, via, dup=True):
    """a shard built on the GPU (the oracle holds its state) or by the oracle (imported by the GPU)"""
    E = _engine()
    kind, metric, d, M, nbits, il = KINDS[name]
    kinds = {"ivf_flat": E.KIND_IVF_FLAT, "ivf_pq": E.KIND_IVF_PQ, "ivf_sq": E.KIND_IVF_SQ16, "ivf_sq8": E.KIND_IVF_SQ8}
    xb = clustered(rs, n, d, ncl=4 * nlist)
    if dup:
        xb[10:14] = xb[3]                     # exact duplicates: equal distances, ties broken by id
    g = E.GpuIndex(kinds[kind], d, metric, nlist=nlist, pq_m=M, pq_nbits=nbits)
    o = S.make_index(kind, d, metric=metric, nlist=nlist, M=M, nbits=nbits)
    if via == "gpu":
        g.set_param("kmeans_niter", _sz(4, 2))
        g.train(xb[: n // 2])
        g.add(xb[: n // 3]); g.add(xb[n // 3:])
        o.set_state(g.get_state())
    else:
        o.train_niter = _sz(4, 2)
        o.train(xb[: n // 2])
        o.add(xb)
        g.set_state(o.get_state())
    if il is not None:
        g.set_param("interleaved", il)
    assert g.ntotal == n == o.ntotal
    return g, o, xb


# ------------------------------------------------------------------ client, CPU
def test_client_accepts_topk_up_to_4096():
    from distributed_faiss_b200.client import IndexClient

    c = IndexClient.__new__(IndexClient)
    assert IndexClient.MAX_TOPK == 4096
    for k in (1, 1025, 4096):
        c._check_topk(k)
    for k in (0, 4097, 3 * 1366):
        with pytest.raises(ValueError, match=f"topk={k}: this engine returns 1..4096 results per query"):
            c._check_topk(k)


# ------------------------------------------------------------------ the gpu tests on the emulator
EMU_SUBSET = [
    "tests/test_ivf_large_k.py::test_large_k_matches_oracle[gpu-flat_ip]",
    "tests/test_ivf_large_k.py::test_large_k_matches_oracle[gpu-sq8]",
    "tests/test_ivf_large_k.py::test_large_k_matches_oracle[oracle-sq16]",
    "tests/test_ivf_large_k.py::test_large_k_matches_oracle[oracle-pq32_interleaved]",
    "tests/test_ivf_large_k.py::test_large_k_matches_oracle[gpu-pq32_row_major]",
    "tests/test_ivf_large_k.py::test_large_k_matches_oracle[oracle-pq24]",
    "tests/test_ivf_large_k.py::test_large_k_matches_oracle[gpu-pq96]",
    "tests/test_ivf_large_k.py::test_large_k_matches_oracle[oracle-pq4_32]",
    "tests/test_ivf_large_k.py::test_large_k_edge_cases[flat_ip]",
    "tests/test_ivf_large_k.py::test_large_k_edge_cases[pq32_interleaved]",
    "tests/test_ivf_large_k.py::test_large_k_search_and_reconstruct",
]
EMU_COUNT = len(EMU_SUBSET)


def test_large_k_gpu_tests_on_the_emulated_library():
    if shutil.which("g++") is None or platform.machine() != "x86_64":
        pytest.skip("the emulator needs g++ on x86-64")
    sys.path.insert(0, os.path.join(ROOT, "tests", "emu"))
    try:
        import build_emu_lib
    finally:
        sys.path.pop(0)
    env = dict(os.environ, DFX_EMU_LIB=build_emu_lib.build())
    run = subprocess.run([sys.executable, "-m", "pytest", "-m", "gpu", "-q", "-x", "-p", "no:cacheprovider"] + EMU_SUBSET,
                         cwd=ROOT, env=env, capture_output=True, text=True, timeout=1500)
    tail = (run.stdout + run.stderr)[-3000:]
    assert run.returncode == 0, tail
    assert f"{EMU_COUNT} passed" in run.stdout, tail


# ------------------------------------------------------------------ GPU parity
@pytest.mark.gpu
@pytest.mark.parametrize("name", list(KINDS))
@pytest.mark.parametrize("via", ["gpu", "oracle"])
def test_large_k_matches_oracle(name, via):
    """every list scan and code layout at k in {1025, 2048, 2049, 4096}: nprobe 1 (padded), several
    probe groups, all lists (filled); duplicate rows keep their id order"""
    kind, metric, d, _, _, _ = KINDS[name]
    rs = np.random.RandomState(1100 + list(KINDS).index(name) + (50 if via == "oracle" else 0))
    nlist = _sz(16, 4)
    n = _sz(6000, 1500)
    g, o, xb = _pair(name, nlist, n, rs, via)
    xq = np.concatenate([clustered(rs, _sz(6, 2), d, ncl=8), xb[3:4]])
    for nprobe in (1, _sz(5, 3), nlist):
        g.nprobe = o.nprobe = nprobe
        for k in KS:
            Dg, Ig = g.search(xq, k)
            Do, Io = o.search(xq, k)
            _assert_same(Dg, Ig, Do, Io, f"{name} via={via} nprobe={nprobe} k={k}")
            assert g.last_stats()["ndis"] == o.last_ndis
        if nprobe == 1:                                    # k > the probed list: padded
            assert (Ig == -1).any() and (Dg[Ig == -1] == _pad_value(kind, metric)).all()
        if nprobe == nlist and n >= 4096:
            assert (Ig >= 0).all()
    row = Ig[-1][Ig[-1] >= 0].tolist()                     # the query is row 3, duplicated at 10..13
    pos = [row.index(i) for i in (3, 10, 11, 12, 13)]
    assert pos == sorted(pos) and np.all(Dg[-1][pos] == Dg[-1][pos[0]])


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["flat_ip", "flat_l2", "pq32_interleaved", "pq4_16"])
def test_large_k_edge_cases(name):
    """few vectors, most lists empty; nprobe 1, 3 and more than nlist; k far above the hits gives
    (FLT_MAX, -1) padding, -FLT_MAX for inner product"""
    kind, metric, d, M, nbits, _ = KINDS[name]
    rs = np.random.RandomState(1200)
    nlist = 8
    xb = clustered(rs, 600, d, ncl=4, sigma=0.05)
    xb[20:25] = xb[0]
    o = S.make_index(kind, d, metric=metric, nlist=nlist, M=M, nbits=nbits)
    o.train_niter = 3
    o.train(xb)
    o.add(xb[np.argsort(((xb - xb[0]) ** 2).sum(1), kind="stable")[:37]])   # one cluster: the other lists stay empty
    E = _engine()
    kinds = {"ivf_flat": E.KIND_IVF_FLAT, "ivf_pq": E.KIND_IVF_PQ}
    g = E.GpuIndex(kinds[kind], d, metric, nlist=nlist, pq_m=M, pq_nbits=nbits)
    g.set_state(o.get_state())
    assert (np.diff(o.list_off) == 0).any()
    for nprobe in (1, 3, 50):
        g.nprobe = o.nprobe = nprobe
        for k in (1025, 4096):
            Dg, Ig = g.search(xb[:9], k)
            Do, Io = o.search(xb[:9], k)
            _assert_same(Dg, Ig, Do, Io, f"{name} edge nprobe={nprobe} k={k}")
            assert g.last_stats()["ndis"] == o.last_ndis
            assert (Ig[:, 37:] == -1).all() and (Dg[Ig == -1] == _pad_value(kind, metric)).all()


@pytest.mark.gpu
def test_large_k_search_and_reconstruct():
    rs = np.random.RandomState(1300)
    nlist = _sz(8, 4)
    g, o, xb = _pair("pq32_interleaved", nlist, _sz(3000, 2100), rs, "oracle", dup=False)
    g.nprobe = o.nprobe = nlist
    Dg, Ig, Rg = g.search_and_reconstruct(xb[:_sz(5, 2)], 2048)
    Do, Io, Ro = o.search_and_reconstruct(xb[:_sz(5, 2)], 2048)
    _assert_same(Dg, Ig, Do, Io, "search_and_reconstruct k=2048")
    assert (Ig >= 0).all() and np.array_equal(Rg, Ro)


@pytest.mark.gpu
@pytest.mark.parametrize("tc", [1, 0])
def test_large_k_both_coarse_paths(tc):
    """nlist 1024: the tensor-core coarse quantizer, and the FFMA one (tensor_cores = 0)"""
    if EMU:
        pytest.skip("1024 lists: too large for the emulator")
    E = _engine()
    rs = np.random.RandomState(1400)
    d, nlist, n = 64, 1024, 100_000
    cent = rs.randn(nlist, d).astype(np.float32)
    xb = (cent[rs.randint(0, nlist, n)] + 0.3 * rs.randn(n, d)).astype(np.float32)
    g = E.GpuIndex(E.KIND_IVF_FLAT, d, L2, nlist=nlist)
    g.set_state({"centroids": cent, "list_off": np.zeros(nlist + 1, np.int64), "ids": np.zeros(0, np.int64),
                 "vecs": np.zeros((0, d), np.float32)})
    g.add(xb)
    o = S.make_index("ivf_flat", d, metric=L2, nlist=nlist)
    o.set_state(g.get_state())
    g.set_param("tensor_cores", tc)
    xq = (cent[rs.randint(0, nlist, 40)] + 0.3 * rs.randn(40, d)).astype(np.float32)
    for nprobe in (8, 64):
        g.nprobe = o.nprobe = nprobe
        for k in (2048, 4096):
            Dg, Ig = g.search(xq, k)
            _assert_same(Dg, Ig, *o.search(xq, k), f"tensor_cores={tc} nprobe={nprobe} k={k}")
            assert g.last_stats()["ndis"] == o.last_ndis


@pytest.mark.gpu
def test_large_k_query_chunks_stay_within_the_budget():
    """the nprobe longest lists bound a candidate row; the query chunk keeps qc x bound composites
    within 128 MiB: a batch of several chunks, compared on the edge rows of every chunk"""
    if EMU:
        pytest.skip("too large for the emulator")
    from tests.test_search_limits import _check_sample, _sample_rows

    E = _engine()
    rs = np.random.RandomState(1500)
    d, nlist, n, k = 32, 64, 400_000, 4096
    cent = rs.randn(nlist, d).astype(np.float32)
    xb = (cent[rs.randint(0, nlist, n)] + 0.3 * rs.randn(n, d)).astype(np.float32)
    g = E.GpuIndex(E.KIND_IVF_FLAT, d, L2, nlist=nlist)
    g.set_state({"centroids": cent, "list_off": np.zeros(nlist + 1, np.int64), "ids": np.zeros(0, np.int64),
                 "vecs": np.zeros((0, d), np.float32)})
    g.add(xb)
    o = S.make_index("ivf_flat", d, metric=L2, nlist=nlist)
    o.set_state(g.get_state())
    nprobe = 48
    g.nprobe = o.nprobe = nprobe
    bound = int(np.sort(np.diff(o.list_off))[::-1][:nprobe].sum())
    chunk = (CAND_BUDGET // 8) // bound
    nq = 3 * chunk + 17
    xq = (cent[rs.randint(0, nlist, nq)] + 0.3 * rs.randn(nq, d)).astype(np.float32)
    D, I = g.search(xq, k)
    assert g.get_param("workspace_bytes") == chunk * bound * 8 <= CAND_BUDGET
    rows = _sample_rows(nq, chunk, rs, extra=8)
    _check_sample(g, xq, k, D, I, rows, o.search, f"k={k} nq={nq} chunk={chunk}")
    assert g.get_param("workspace_bytes") <= CAND_BUDGET


@pytest.mark.gpu
def test_large_k_refuses_a_list_over_the_budget():
    """one probed list of 2^24 + 1 vectors: its candidates alone exceed 128 MiB; the search raises
    before it launches anything, and k <= 1024 still searches the shard"""
    if EMU:
        pytest.skip("2^24 vectors: too large for the emulator")
    E = _engine()
    rs = np.random.RandomState(1600)
    d, M, nlist, big = 4, 4, 2, (1 << 24) + 1
    g = E.GpuIndex(E.KIND_IVF_PQ, d, L2, nlist=nlist, pq_m=M)
    g.set_state({"centroids": np.array([[0, 0, 0, 0], [100, 100, 100, 100]], np.float32),
                 "codebooks": rs.randn(M, 256, 1).astype(np.float32),
                 "list_off": np.array([0, big, big + 3], np.int64), "ids": np.arange(big + 3, dtype=np.int64),
                 "codes": rs.randint(0, 256, (big + 3, M)).astype(np.uint8)})
    xq = np.zeros((2, d), np.float32)
    g.nprobe = 1
    before = E.launch_count()
    with pytest.raises(RuntimeError, match=r"IVF search at k=2048 with nprobe=1: one query's candidates can reach "
                                           r"16777217 vectors"):
        g.search(xq, 2048)
    assert E.launch_count() == before
    D, I = g.search(xq, 10)
    assert (I >= 0).all() and (I < big).all()
    g.nprobe = 2
    with pytest.raises(RuntimeError, match="nprobe=2: one query's candidates can reach 16777220 vectors"):
        g.search(xq, 1025)


# ------------------------------------------------------------------ two knnlm servers, end to end
@pytest.mark.gpu
def test_knnlm_large_k_through_the_client_over_sockets_and_the_plane():
    """IndexClient.search(topk=2000) and search_with_filter(top_k=1000), which asks every shard for
    3000: the merge of the oracle's answers on each server's shard, over the socket fan-out and over
    the search plane"""
    if EMU:
        pytest.skip("CUDA tensors")
    from distributed_faiss_b200.index_cfg import IndexCfg
    from oracle import oracle as O
    from tests.test_gpu_api import _plane_cluster, wait_trained

    store, servers, plane, client = _plane_cluster(2)
    try:
        rs = np.random.RandomState(1700)
        d, nlist, M, nprobe = 128, 8, 32, 8
        cfg = IndexCfg(index_builder_type="knnlm", dim=d, centroids=nlist, metric="l2", train_num=2000, code_size=M)
        client.create_index("kn", cfg)
        nxt = 0
        for b in range(8):
            x = clustered(rs, 1100, d, ncl=8)
            client.add_index_data("kn", x, [(i, i % 3) for i in range(nxt, nxt + 1100)], False)
            nxt += 1100
        client.sync_train("kn")
        wait_trained(client, "kn")
        import time

        t0 = time.time()
        while client.get_ntotal("kn") != nxt:
            assert time.time() - t0 < 300, "adds never finished"
            time.sleep(0.05)
        client.set_nprobe("kn", nprobe)
        xq = clustered(rs, 12, d, ncl=8)

        def oracle_merge(k):
            Ds, Is, metas = [], [], []
            for s in servers:
                ix = s.indexes["kn"]
                o = O.make_index("ivf_pq", d, metric=L2, nlist=nlist, M=M)
                o.set_state(ix.faiss_index.get_state())
                o.nprobe = nprobe
                Do, Io = o.search(xq, k)
                Dg, Ig = ix.faiss_index.search(xq, k)
                _assert_same(Dg, Ig, Do, Io, f"shard {s} k={k}")
                Ds.append(Do); Is.append(Io); metas.append(ix.id_to_metadata)
            Dall = np.stack(Ds)
            pos = np.arange(Dall.size, dtype=np.int64).reshape(Dall.shape)
            refD, refP = O.merge(Dall, pos)
            S_, nq_, k_ = Dall.shape
            meta = [[metas[p // (nq_ * k_)][int(Is[p // (nq_ * k_)][q, p % k_])] for p in refP[q]] for q in range(nq_)]
            return refD, meta

        refD, refM = oracle_merge(2000)
        for path in ("plane", "sockets"):
            if path == "sockets":
                client.detach_plane()
            D, meta = client.search(xq, 2000, "kn")
            assert np.array_equal(np.asarray(D, dtype=np.float32), refD), path
            assert [list(r) for r in meta] == refM, path
            client.plane = plane

        refD3, refM3 = oracle_merge(3000)
        for fv in (0, 2):
            want = []
            for q in range(len(xq)):
                kept = [(s, m) for s, m in zip(refD3[q], refM3[q]) if m[1] != fv][:1000]
                want.append(kept)
            for path in ("plane", "sockets"):
                if path == "sockets":
                    client.detach_plane()
                scores, meta = client.search_with_filter(xq, 1000, "kn", filter_pos=1, filter_value=fv)
                for q in range(len(xq)):
                    assert list(meta[q]) == [m for _, m in want[q]], (path, fv, q)
                    assert np.array_equal(np.asarray(scores[q], np.float32).reshape(-1),
                                          np.array([s for s, _ in want[q]], np.float32)), (path, fv, q)
                client.plane = plane
    finally:
        client.close()
        plane.stop()
        for s in servers:
            s.stop()
