"""IVF-PQ with 4-bit codes (knnlm with bits_per_vector=4): the packed code layout, the shuffle-lookup
list scan (dfx_scan_pq4_dev.cuh) and the build path at 16 centroids per sub-quantizer.

CPU: the faiss file format at nbits = 4, persistence and sharded search through the servers with
oracle engines, and this file's `gpu` tests run against the emulated library.
GPU: the CUDA kernels against the oracle, bit for bit (distances, ids, ndis, codes, t-values,
reconstruction), the device-resident and graph-captured paths, and the servers / client end to end."""
import os
import platform
import shutil
import struct
import subprocess
import sys
import tempfile
import threading

import numpy as np
import pytest

from tests.conftest import clustered

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
IP, L2 = 0, 1
FMAX = np.finfo(np.float32).max
EMU = bool(os.environ.get("DFX_EMU_LIB"))


def _sz(full, emu):
    return emu if EMU else full


def _oracle4(d, nlist, M, n, rs, metric=L2, niter=4):
    from oracle import oracle as O

    o = O.make_index("ivf_pq", d, metric=metric, nlist=nlist, M=M, nbits=4)
    o.train_niter = niter
    xb = clustered(rs, n, d, ncl=max(4, nlist // 2))
    o.train(xb); o.add(xb)
    return o, xb


# ------------------------------------------------------------------ faiss file format, CPU
def test_pq4_faiss_file_roundtrip_and_layout(oracle_lib, tmp_path):
    from distributed_faiss_b200 import faiss_io

    rs = np.random.RandomState(3)
    d, nlist, M, n = 64, 4, 16, 300
    o, _ = _oracle4(d, nlist, M, n, rs)
    st = o.get_state()
    assert st["ksub"] == 16 and st["codes"].max() < 16
    st["codes"][0, :2] = (3, 12)                                       # known answer: byte 0xC3
    path = str(tmp_path / "pq4.faiss")
    faiss_io.write_index(st, path, nprobe=2)
    st2, nprobe = faiss_io.read_index(path)
    assert nprobe == 2 and st2["kind"] == "ivf_pq" and st2["M"] == M and st2["ksub"] == 16
    assert st2["codes"].shape == (n, M) and st2["codebooks"].shape == (M, 16, d // M)
    for key in ("centroids", "codebooks", "list_off", "ids", "codes"):
        assert np.asarray(st2[key]).tobytes() == np.asarray(st[key]).tobytes(), key
    raw = open(path, "rb").read()
    assert raw[:4] == b"IwPQ"
    off = 4 + 33 + 16 + 4 + 33 + 8 + 4 * nlist * d + 9
    assert struct.unpack_from("<BQQQQ", raw, off) == (1, M // 2, d, M, 4)  # by_residual, code_size, pq.d, pq.M, nbits
    off += 33
    assert struct.unpack_from("<Q", raw, off) == (M * 16 * (d // M),)       # codebook floats
    off += 8 + 4 * M * 16 * (d // M)
    assert raw[off:off + 4] == b"ilar" and struct.unpack_from("<QQ", raw, off + 4) == (nlist, M // 2)
    sizes = np.diff(st["list_off"])
    assert raw[off + 20:off + 24] == b"full"
    first = off + 24 + 8 + 8 * nlist                                      # codes of the first non-empty list
    assert sizes[0] > 0 and raw[first] == 0xC3
    assert len(raw) == first + n * (M // 2 + 8)


def test_pq4_faiss_file_rejects_other_bit_widths(oracle_lib, tmp_path):
    from distributed_faiss_b200 import faiss_io

    rs = np.random.RandomState(4)
    o, _ = _oracle4(32, 4, 8, 200, rs)
    st = o.get_state()
    with pytest.raises(faiss_io.FaissFormatError, match="8-bit and 4-bit"):
        faiss_io.write_index(dict(st, ksub=64), str(tmp_path / "x.faiss"))
    path = str(tmp_path / "pq4.faiss")
    faiss_io.write_index(st, path)
    raw = bytearray(open(path, "rb").read())
    off = 4 + 33 + 16 + 4 + 33 + 8 + 4 * 4 * 32 + 9 + 1 + 8 + 16          # pq.nbits
    assert struct.unpack_from("<Q", raw, off) == (4,)
    struct.pack_into("<Q", raw, off, 6)
    open(path, "wb").write(bytes(raw))
    with pytest.raises(faiss_io.FaissFormatError, match="8 or 4 bits"):
        faiss_io.read_index(path)


# ------------------------------------------------------------------ persistence / servers, CPU
def _knnlm4(d, nlist, M, **kw):
    from distributed_faiss_b200.index_cfg import IndexCfg

    return IndexCfg(index_builder_type="knnlm", dim=d, centroids=nlist, metric="l2", code_size=M,
                    bits_per_vector=4, **kw)


def _wait_trained_index(ix):
    import time

    from distributed_faiss_b200.index_state import IndexState

    t0 = time.time()
    while ix.get_state() != IndexState.TRAINED:
        assert time.time() - t0 < 60, "index never reached TRAINED"
        time.sleep(0.01)


@pytest.mark.parametrize("fmt", ["dfx", "faiss"])
def test_pq4_shard_saved_and_loaded(oracle_lib, tmp_path, fmt):
    from distributed_faiss_b200.index import Index
    from distributed_faiss_b200.index_cfg import IndexCfg
    from tests.oracle_engine import oracle_engine_factory

    rs = np.random.RandomState(5)
    d, nlist, M = 32, 6, 16
    cfg = _knnlm4(d, nlist, M, train_num=400, index_storage_dir=str(tmp_path), index_format=fmt)
    ix = Index(cfg, engine_factory=oracle_engine_factory)
    x = clustered(rs, 500, d, ncl=6)
    ix.add_batch(x, [("m", i) for i in range(500)], train_async_if_triggered=False)
    ix.train()
    _wait_trained_index(ix)
    assert ix.faiss_index.ksub == 16
    ix.set_nprobe(3)
    assert ix.save()
    q = x[::50] + np.float32(0.01)
    D1, m1, _ = ix.search(q, 7)
    cfg2 = IndexCfg.from_json(str(tmp_path / "cfg.json"))
    assert cfg2.extra["bits_per_vector"] == 4
    ix2 = Index.from_storage_dir(str(tmp_path), cfg2, engine_factory=oracle_engine_factory)
    ix2.set_nprobe(3)
    a, b = ix.faiss_index.get_state(), ix2.faiss_index.get_state()
    for key in ("centroids", "codebooks", "list_off", "ids", "codes", "tvals"):
        assert np.asarray(a[key]).tobytes() == np.asarray(b[key]).tobytes(), key
    D2, m2, _ = ix2.search(q, 7)
    assert D1.tobytes() == D2.tobytes() and m1 == m2
    # the same files under a cfg that builds other codes are refused, naming both shapes
    for other in (dict(bits_per_vector=8), dict(code_size=8)):
        bad = _knnlm4(d, nlist, M, index_format=fmt)
        bad.extra.update(other)
        with pytest.raises(RuntimeError, match=r"\(M, ksub\) = \(16, 16\)"):
            Index.from_storage_dir(str(tmp_path), bad, engine_factory=oracle_engine_factory)


def test_pq4_sharded_search_is_the_merge_of_the_shards(oracle_lib):
    from distributed_faiss_b200.client import ResultHeap
    from distributed_faiss_b200.index_state import IndexState
    from distributed_faiss_b200.server import IndexServer
    from oracle import oracle as O
    from tests.oracle_engine import oracle_engine_factory, oracle_merge
    from tests.test_host_logic import free_ports, make_client, wait_listening, wait_trained

    ResultHeap.merge_backend = staticmethod(oracle_merge)
    tmp = tempfile.TemporaryDirectory()
    ports = free_ports(2)
    servers = [IndexServer(r, tmp.name, engine_factory=oracle_engine_factory) for r in range(2)]
    for s, p in zip(servers, ports):
        threading.Thread(target=s.start_blocking, args=(p,), daemon=True).start()
    wait_listening(ports)
    try:
        rs = np.random.RandomState(6)
        d, nlist, M, k = 64, 8, 32, 12
        client = make_client(ports)
        client.create_index("pq4", _knnlm4(d, nlist, M, train_num=600))
        xs = [clustered(rs, 400, d, ncl=8) for _ in range(4)]
        for b, x in enumerate(xs):
            client.add_index_data("pq4", x, list(range(400 * b, 400 * (b + 1))), False)
        client.sync_train("pq4")
        wait_trained(client, "pq4")
        import time

        t0 = time.time()
        while client.get_ntotal("pq4") != 1600 or client.get_state("pq4") != IndexState.TRAINED:
            assert time.time() - t0 < 60, "adds never finished"
            time.sleep(0.02)
        client.set_nprobe("pq4", 3)
        xq = np.concatenate(xs)[::101][:12] + np.float32(0.01)
        D, meta = client.search(xq, k, "pq4")
        Ds, Ps, metas = [], [], []
        for s in servers:
            ix = s.indexes["pq4"]
            assert ix.faiss_index.ksub == 16 and ix.faiss_index.M == M
            Do, Io = ix.faiss_index.search(xq, k)
            Ds.append(Do); Ps.append(Io); metas.append(ix.id_to_metadata)
        Dall = np.stack(Ds)
        pos = np.arange(Dall.size, dtype=np.int64).reshape(Dall.shape)
        refD, refP = O.merge(Dall, pos)
        assert np.array_equal(np.asarray(D, dtype=np.float32), refD)
        S_, nq_, k_ = Dall.shape
        want = [[metas[p // (nq_ * k_)][int(Ps[p // (nq_ * k_)][q, p % k_])] for p in refP[q]] for q in range(nq_)]
        assert [list(r) for r in meta] == want
        client.close()
    finally:
        for s in servers:
            s.stop()


# ------------------------------------------------------------------ the gpu tests on the emulator
EMU_SUBSET = [
    "tests/test_ivf_pq4.py::test_pq4_matches_oracle[gpu-128-32-1]",
    "tests/test_ivf_pq4.py::test_pq4_matches_oracle[oracle-96-24-1]",
    "tests/test_ivf_pq4.py::test_pq4_matches_oracle[oracle-128-128-1]",
    "tests/test_ivf_pq4.py::test_pq4_matches_oracle[gpu-128-32-0]",
    "tests/test_ivf_pq4.py::test_pq4_edge_cases",
    "tests/test_ivf_pq4.py::test_pq4_reconstruct_matches_oracle",
    "tests/test_ivf_pq4.py::test_pq4_m32_is_never_interleaved",
    "tests/test_ivf_pq4.py::test_pq4_limits",
]


def test_pq4_gpu_tests_on_the_emulated_library():
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
    assert f"{len(EMU_SUBSET)} passed" in run.stdout, tail


# ------------------------------------------------------------------ GPU parity
def _assert_same(Dg, Ig, Do, Io, what):
    if not (np.array_equal(Ig, Io) and np.array_equal(Dg, Do)):
        bad = np.argwhere((Ig != Io) | (Dg != Do))
        q, j = bad[0]
        raise AssertionError(f"{what}: {len(bad)} mismatching slots of {Ig.size}; first at q={q} j={j}: "
                             f"gpu=({Dg[q, j]!r},{Ig[q, j]}) oracle=({Do[q, j]!r},{Io[q, j]})")


def _pair(d, nlist, M, metric=L2):
    from distributed_faiss_b200 import engine as E
    from oracle import oracle as O

    return (E.GpuIndex(E.KIND_IVF_PQ, d, metric, nlist=nlist, pq_m=M, pq_nbits=4),
            O.make_index("ivf_pq", d, metric=metric, nlist=nlist, M=M, nbits=4))


def _check_gpu_build(st, o, xb, metric):
    """device encoding: a shard trained and filled on the GPU holds the oracle's codes and t-values
    of the same rows under the same centroids and codebooks"""
    from oracle import oracle as O

    lists = O.assign(metric, st["centroids"], xb)
    order = np.argsort(lists, kind="stable")
    assert np.array_equal(st["ids"], order)
    enc = o._encode(xb[order], lists[order])
    assert st["codes"].max() < 16
    assert st["codes"].tobytes() == enc["codes"].tobytes()
    assert st["tvals"].tobytes() == enc["tvals"].tobytes()


def _build_both(d, nlist, M, n, rs, via, metric=L2, niter=None):
    xb = clustered(rs, n, d, ncl=max(8, nlist // 2))
    g, o = _pair(d, nlist, M, metric)
    if via == "gpu":
        if niter or EMU:
            g.set_param("kmeans_niter", niter or 2)
        g.train(xb[: n // 2])
        g.add(xb[: n // 3]); g.add(xb[n // 3:])
        st = g.get_state()
        assert st["ksub"] == 16 and st["codebooks"].shape == (M, 16, d // M)
        o.set_state(st)
        _check_gpu_build(st, o, xb, metric)
    else:
        o.train_niter = 4
        o.train(xb[: n // 2])
        o.add(xb)
        g.set_state(o.get_state())
        assert np.array_equal(g.get_array("tvals"), o.tvals)
        assert np.array_equal(g.get_array("codes").reshape(-1, M), o.codes)
    assert g.ntotal == n == o.ntotal
    return g, o, xb


@pytest.mark.gpu
@pytest.mark.parametrize("d,M,metric", [(128, 8, L2), (128, 16, L2), (128, 32, L2), (128, 64, L2), (128, 128, L2),
                                        (96, 24, L2), (768, 96, L2), (128, 32, IP)])
@pytest.mark.parametrize("via", ["gpu", "oracle"])
def test_pq4_matches_oracle(d, M, metric, via):
    """distances, ids and ndis bit for bit; metric = the coarse quantizer's (knnlm with metric="dot"
    probes by inner product and scans by L2, quirk B2)"""
    rs = np.random.RandomState(10)
    nlist = 16
    g, o, xb = _build_both(d, nlist, M, _sz(6000, 1200), rs, via, metric)
    xq = np.concatenate([clustered(rs, _sz(20, 4), d, ncl=8), xb[:3] + 0.01 * rs.randn(3, d).astype(np.float32)])
    for nprobe in (nlist, 1, 5):   # all lists; one; several probe groups per query
        g.nprobe = nprobe; o.nprobe = nprobe
        for k in ((1, 10, 100, 300, 1024) if not EMU else (10, 1024)):   # 1024 > hits at nprobe 1
            Dg, Ig = g.search(xq, k)
            Do, Io = o.search(xq, k)
            _assert_same(Dg, Ig, Do, Io, f"M={M} d={d} metric={metric} via={via} nprobe={nprobe} k={k}")
            assert g.last_stats()["ndis"] == o.last_ndis
        if nprobe == 1:
            assert (Ig == -1).any() and (Dg[Ig == -1] == FMAX).all()


@pytest.mark.gpu
def test_pq4_edge_cases():
    """empty and single-vector lists, lists whose length is not a multiple of 32, exact duplicates
    (ties broken by id), k > hits, nprobe > nlist"""
    from oracle import oracle as O

    rs = np.random.RandomState(11)
    d, nlist, M = 64, 8, 16
    xb = clustered(rs, 600, d, ncl=4, sigma=0.05)
    xb[10:20] = xb[0]
    o = O.make_index("ivf_pq", d, metric=L2, nlist=nlist, M=M, nbits=4)
    o.train_niter = 4
    o.train(xb)
    far = (100.0 + rs.randn(1, d)).astype(np.float32)
    o.centroids[-1] = far[0]                                    # the last list holds `far` alone
    o.add(np.concatenate([xb[:37], far]))
    sizes = np.diff(o.list_off)
    assert sizes[-1] == 1 and (sizes == 0).any() and (sizes % 32 != 0).any()
    g, _ = _pair(d, nlist, M)
    g.set_state(o.get_state())
    xq = np.concatenate([xb[:9], far])
    for nprobe in (1, 3, 50):
        g.nprobe = nprobe; o.nprobe = nprobe
        for k in (1, 64):
            Dg, Ig = g.search(xq, k)
            Do, Io = o.search(xq, k)
            _assert_same(Dg, Ig, Do, Io, f"edge nprobe={nprobe} k={k}")
            assert g.last_stats()["ndis"] == o.last_ndis
        assert (Ig == -1).any() and (Dg[Ig == -1] == FMAX).all()
    assert Ig[-1][0] == 37                                        # the lone vector finds itself
    row = Ig[0][Ig[0] >= 0].tolist()
    pos = [row.index(i) for i in [0] + list(range(10, 20))]
    assert pos == sorted(pos) and np.all(Dg[0][pos] == Dg[0][pos[0]])   # equal distances, ascending ids


@pytest.mark.gpu
def test_pq4_reconstruct_matches_oracle():
    rs = np.random.RandomState(14)
    g, o, xb = _build_both(128, 8, 32, _sz(3000, 800), rs, "oracle")
    ids = np.array([0, 5, len(xb) - 1, -1, 17], dtype=np.int64)
    R_g, R_o = g.reconstruct_rows(ids), o.reconstruct_rows(ids)
    assert np.isnan(R_g[3]).all()
    assert np.array_equal(R_g[[0, 1, 2, 4]], R_o[[0, 1, 2, 4]])
    g.nprobe = o.nprobe = 4
    Dg, Ig, Rg = g.search_and_reconstruct(xb[:6], 5)
    Do, Io, Ro = o.search_and_reconstruct(xb[:6], 5)
    _assert_same(Dg, Ig, Do, Io, "search_and_reconstruct")
    assert np.array_equal(Rg, Ro)


@pytest.mark.gpu
def test_pq4_m32_is_never_interleaved():
    """the interleaved M = 32 layout holds one byte per code: a 4-bit M = 32 shard stays row-major,
    whatever the `interleaved` knob says, and answers the same"""
    rs = np.random.RandomState(15)
    g, o, xb = _build_both(128, 8, 32, _sz(2000, 600), rs, "oracle")
    xq = xb[:5] + np.float32(0.01)
    g.nprobe = o.nprobe = 3
    D0, I0 = g.search(xq, 10)
    for il in (0, 1):
        g.set_param("interleaved", il)
        D1, I1 = g.search(xq, 10)
        _assert_same(D1, I1, D0, I0, f"interleaved={il}")
        assert np.array_equal(g.get_array("codes").reshape(-1, 32), o.codes)
    Do, Io = o.search(xq, 10)
    _assert_same(D0, I0, Do, Io, "interleaved")


@pytest.mark.gpu
def test_pq4_limits():
    from distributed_faiss_b200 import engine as E

    for M, d in ((8, 64), (24, 96), (128, 256)):
        E.GpuIndex(E.KIND_IVF_PQ, d, L2, nlist=4, pq_m=M, pq_nbits=4)
    for M, d in ((4, 64), (12, 96), (136, 272), (20, 100)):
        with pytest.raises(RuntimeError, match=r"multiple of 8 in \[8, 128\] that divides d"):
            E.GpuIndex(E.KIND_IVF_PQ, d, L2, nlist=4, pq_m=M, pq_nbits=4)
    for nbits in (2, 6, 16):
        with pytest.raises(RuntimeError, match="8 or 4 bits per sub-quantizer"):
            E.GpuIndex(E.KIND_IVF_PQ, 64, L2, nlist=4, pq_m=8, pq_nbits=nbits)
    # codes arrive one per byte and must fit in 4 bits
    rs = np.random.RandomState(16)
    o, _ = _oracle4(64, 4, 8, 200, rs)
    st = o.get_state()
    g, _ = _pair(64, 4, 8)
    bad = st["codes"].copy()
    bad[7, 3] = 16
    with pytest.raises(RuntimeError, match=r"4-bit code must be in \[0, 16\)"):
        g.set_state(dict(st, codes=bad))


@pytest.mark.gpu
def test_pq4_device_paths_match_the_host_path(monkeypatch):
    """search_dev equals search; a ShardGroup of 4-bit shards replays its search from a captured
    CUDA graph with the eager answers"""
    if EMU:
        pytest.skip("CUDA tensors")
    import torch

    from distributed_faiss_b200 import spmd

    rs = np.random.RandomState(17)
    shards, tables, base = [], [], 0
    for s in range(2):
        g, o, xb = _build_both(128, 32, 64 if s == 0 else 32, 8000, rs, "gpu")
        g.nprobe = 6
        shards.append(g)
        tables.append(torch.arange(base, base + 8000, dtype=torch.int64, device="cuda"))
        base += 8000
    xq = np.concatenate([clustered(rs, 40, 128, ncl=8), xb[:8] + np.float32(0.01)])
    x_t = torch.from_numpy(xq).cuda()
    for g in shards:
        D, I = g.search(xq, 20)
        Dd, Id = g.search_dev(x_t, 20)
        torch.cuda.synchronize()
        assert np.array_equal(Dd.cpu().numpy(), D) and np.array_equal(Id.cpu().numpy(), I)
    graphed = spmd.ShardGroup(shards, tables)
    monkeypatch.setenv("DFX_GRAPHS", "0")
    eager = spmd.ShardGroup(shards, tables)
    D0, I0 = eager.search(x_t, 20)
    for _ in range(3):   # capture, then replays
        D1, I1 = graphed.search(x_t, 20)
        assert torch.equal(I0, I1) and torch.equal(D0, D1)
    assert graphed._graph_max_nq > 0 and len(graphed._graphs) == 1   # the capture did not fall back to eager


@pytest.mark.gpu
def test_pq4_gpu_training_quality():
    """GPU-trained 4-bit codes reconstruct the data within 1.25x the oracle's error, on the data and
    bound of the 8-bit test_gpu_training_quality (the two trainings sample differently, so they are
    not bit-comparable)"""
    if EMU:
        pytest.skip("too large for the emulator")
    rs = np.random.RandomState(9)
    d, nlist, M, n = 64, 32, 16, 20000
    xb = clustered(rs, n, d, ncl=40, sigma=0.2)
    g, o = _pair(d, nlist, M)
    g.train(xb); g.add(xb)
    o.train(xb); o.add(xb)
    ids = np.arange(0, n, 7, dtype=np.int64)
    err_g = float(((g.reconstruct_rows(ids) - xb[::7]) ** 2).sum(1).mean())
    err_o = float(((o.reconstruct_rows(ids) - xb[::7]) ** 2).sum(1).mean())
    assert err_g < 1.25 * err_o + 1e-6, (err_g, err_o)


def _start_servers(n, root):
    from distributed_faiss_b200.server import IndexServer
    from tests.test_gpu_api import free_ports, wait_listening

    ports = free_ports(n)
    servers = [IndexServer(r, root) for r in range(n)]
    for s, p in zip(servers, ports):
        threading.Thread(target=s.start_blocking, args=(p,), daemon=True).start()
    wait_listening(ports)
    return servers, ports


def _wait_ntotal(client, index_id, n):
    import time

    from distributed_faiss_b200.index_state import IndexState

    t0 = time.time()
    while client.get_ntotal(index_id) != n or client.get_state(index_id) != IndexState.TRAINED:
        assert time.time() - t0 < 300, "adds never finished"
        time.sleep(0.05)


@pytest.mark.gpu
def test_knnlm_4bit_sharded_through_the_client_with_embeddings_and_faiss_files():
    """two IndexServers on the GPU engine, knnlm with bits_per_vector=4: the client's merged answer
    (with return_embeddings) is the merge of the oracle's answers on each shard, and a save in faiss
    format loads back into the same state and answers"""
    if EMU:
        pytest.skip("CUDA tensors")
    from distributed_faiss_b200.index_cfg import IndexCfg
    from oracle import oracle as O
    from tests.test_gpu_api import make_client

    tmp = tempfile.TemporaryDirectory()
    servers, ports = _start_servers(2, tmp.name)
    try:
        rs = np.random.RandomState(19)
        d, nlist, M, k, index_id = 128, 8, 32, 20, "pq4"
        client = make_client(ports)
        cfg = IndexCfg(index_builder_type="knnlm", dim=d, centroids=nlist, metric="l2", train_num=1000, code_size=M,
                       bits_per_vector=4, index_format="faiss")
        client.create_index(index_id, cfg)
        xs = [clustered(rs, 1000, d, ncl=8) for _ in range(4)]
        for b, x in enumerate(xs):
            client.add_index_data(index_id, x, list(range(1000 * b, 1000 * (b + 1))), False)
        client.sync_train(index_id)
        _wait_ntotal(client, index_id, 4000)
        client.set_nprobe(index_id, 3)
        xq = np.concatenate(xs)[::211][:16] + np.float32(0.01)
        D, meta, embs = client.search(xq, k, index_id, return_embeddings=True)
        Ds, Ps, Rs, metas, before = [], [], [], [], []
        for s in servers:
            ix = s.indexes[index_id]
            assert ix.faiss_index.pq_nbits == 4 and ix.faiss_index.nprobe == 3
            st = ix.faiss_index.get_state()
            before.append(st)
            o = O.make_index("ivf_pq", d, metric=L2, nlist=nlist, M=M, nbits=4)
            o.set_state(st)
            o.nprobe = 3
            Do, Io, Ro = o.search_and_reconstruct(xq, k)
            Ds.append(Do); Ps.append(Io); Rs.append(Ro); metas.append(ix.id_to_metadata)
        Dall = np.stack(Ds)
        pos = np.arange(Dall.size, dtype=np.int64).reshape(Dall.shape)
        refD, refP = O.merge(Dall, pos)
        assert np.array_equal(np.asarray(D, dtype=np.float32), refD)
        S_, nq_, k_ = Dall.shape
        want = [[metas[p // (nq_ * k_)][int(Ps[p // (nq_ * k_)][q, p % k_])] for p in refP[q]] for q in range(nq_)]
        assert [list(r) for r in meta] == want
        for q in range(nq_):
            for j, p in enumerate(refP[q]):
                s_, jj = p // (nq_ * k_), p % k_
                assert np.array_equal(np.asarray(embs[q][j], dtype=np.float32), Rs[s_][q, jj])
        client.save_index(index_id)
        assert os.path.isfile(os.path.join(tmp.name, index_id, "0", "index.faiss"))
        client.drop_index(index_id)
        client.close()
        c2 = make_client(ports)
        assert c2.load_index(index_id, cfg)
        c2.set_nprobe(index_id, 3)
        for s, st in zip(servers, before):
            after = s.indexes[index_id].faiss_index.get_state()
            for key in ("centroids", "codebooks", "list_off", "ids", "codes", "tvals"):
                assert np.asarray(after[key]).tobytes() == np.asarray(st[key]).tobytes(), key
        D1, M1 = c2.search(xq, k, index_id)
        assert np.array_equal(np.asarray(D1, dtype=np.float32), refD) and M1 == meta
        c2.close()
    finally:
        for s in servers:
            s.stop()
