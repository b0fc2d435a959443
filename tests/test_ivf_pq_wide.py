"""IVF-PQ with 65 to 128 sub-quantizers (knnlm code_size / "IVF{n},PQ{M}" with 64 < M <= 128):
the wide-code list scan (dfx_scan_pq_wide_dev.cuh) and the build path at that width.

CPU: the factory and builder limits, the oracle against the float64 restatement, the faiss file
format, and this file's `gpu` tests run against the emulated library.
GPU: the CUDA kernels against the oracle, bit for bit (distances, ids, ndis, codes, t-values,
reconstruction), and the servers / client / faiss-file paths end to end."""
import os
import platform
import shutil
import struct
import subprocess
import sys

import numpy as np
import pytest

from tests.conftest import clustered

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
L2 = 1
FMAX = np.finfo(np.float32).max
EMU = bool(os.environ.get("DFX_EMU_LIB"))


def _sz(full, emu):
    return emu if EMU else full


# ------------------------------------------------------------------ limits, CPU
@pytest.mark.parametrize("d,s,M", [(768, "IVF64,PQ96", 96), (768, "IVF64,PQ128x8", 128), (640, "IVF32,PQ80", 80),
                                   (1024, "IVF64,PQ128", 128)])
def test_factory_accepts_up_to_128_sub_quantizers(d, s, M):
    from distributed_faiss_b200.factory import FactorySpec, parse_factory

    assert parse_factory(d, s, L2) == FactorySpec("ivf_pq", L2, int(s[3:s.index(",")]), M)


@pytest.mark.parametrize("s", ["IVF64,PQ132", "IVF64,PQ256"])
def test_factory_rejects_more_than_128_sub_quantizers(s):
    from distributed_faiss_b200.factory import parse_factory

    with pytest.raises(RuntimeError, match="sub-quantizers must be a multiple of 4, at most 128, that divides d=768"):
        parse_factory(768, s, L2)


def test_knnlm_code_size_96_reaches_the_engine(monkeypatch):
    from distributed_faiss_b200 import engine
    from distributed_faiss_b200.index import default_engine_factory
    from distributed_faiss_b200.index_cfg import IndexCfg

    made = []

    class Recorder:
        nprobe = 1

        def __init__(self, kind, d, metric, **kw):
            made.append((kind, d, metric, kw))

    monkeypatch.setattr(engine, "GpuIndex", Recorder)
    default_engine_factory(IndexCfg(index_builder_type="knnlm", dim=768, centroids=64, metric="l2", code_size=96))
    (kind, d, metric, kw), = made
    assert kind == engine.KIND_IVF_PQ and d == 768 and metric == L2
    assert kw["pq_m"] == 96 and kw["pq_nbits"] == 8 and kw["nlist"] == 64


# ------------------------------------------------------------------ oracle, CPU
@pytest.mark.parametrize("d,M", [(384, 96), (512, 128)])
def test_wide_pq_oracle_close_to_float64(oracle_lib, d, M):
    from oracle import oracle as O
    from oracle import ref_numpy as R

    rs = np.random.RandomState(2)
    nlist = 8
    xb = clustered(rs, 3000, d, ncl=nlist)
    o = O.make_index("ivf_pq", d, metric=L2, nlist=nlist, M=M)
    o.train_niter = 6
    o.train(xb[:1500]); o.add(xb)
    xq = clustered(rs, 16, d, ncl=8)
    for nprobe in (nlist, 3):
        o.nprobe = nprobe
        Do, Io = o.search(xq, 10)
        D64, I64 = R.ivf_search(o.get_state(), xq, nprobe, 10)
        scale = (xq.astype(np.float64) ** 2).sum(1, keepdims=True) + (xb.astype(np.float64) ** 2).sum(1).max()
        assert (np.abs(Do - D64) <= 1e-4 * scale).all()
        gap = np.abs(np.diff(D64, axis=1))
        sep = np.ones_like(Io, dtype=bool)
        sep[:, 1:] &= gap > 1e-5 * scale
        sep[:, :-1] &= gap > 1e-5 * scale
        assert np.array_equal(Io[sep], I64[sep])


def test_wide_pq_faiss_file_roundtrip_and_layout(oracle_lib, tmp_path):
    from distributed_faiss_b200 import faiss_io
    from oracle import oracle as O

    rs = np.random.RandomState(3)
    d, nlist, M, n = 192, 4, 96, 400
    o = O.make_index("ivf_pq", d, metric=L2, nlist=nlist, M=M)
    o.train_niter = 4
    xb = clustered(rs, n, d, ncl=4)
    o.train(xb); o.add(xb)
    st = o.get_state()
    path = str(tmp_path / "pq96.faiss")
    faiss_io.write_index(st, path, nprobe=2)
    st2, nprobe = faiss_io.read_index(path)
    assert nprobe == 2 and st2["kind"] == "ivf_pq" and st2["M"] == M and st2["codes"].shape == (n, M)
    for key in ("centroids", "codebooks", "list_off", "ids", "codes"):
        assert np.asarray(st2[key]).tobytes() == np.asarray(st[key]).tobytes(), key
    raw = open(path, "rb").read()
    assert raw[:4] == b"IwPQ"
    assert struct.unpack_from("<iqqqBi", raw, 4) == (d, n, 1 << 20, 1 << 20, 1, L2)
    off = 4 + 33 + 16
    assert raw[off:off + 4] == b"IxF2"                                   # L2 coarse quantizer
    off += 4 + 33 + 8 + 4 * nlist * d + 9
    assert struct.unpack_from("<BQQQQ", raw, off) == (1, M, d, M, 8)     # by_residual, code_size, pq.d, pq.M, nbits
    off += 33
    assert struct.unpack_from("<Q", raw, off) == (M * 256 * (d // M),)   # codebook floats
    off += 8 + 4 * M * 256 * (d // M)
    assert raw[off:off + 4] == b"ilar" and struct.unpack_from("<QQ", raw, off + 4) == (nlist, M)   # code_size = M
    assert len(raw) == off + 24 + 8 + 8 * nlist + n * (M + 8)


# ------------------------------------------------------------------ the gpu tests on the emulator
EMU_SUBSET = [
    "tests/test_ivf_pq_wide.py::test_wide_pq_matches_oracle[oracle-272-68]",
    "tests/test_ivf_pq_wide.py::test_wide_pq_matches_oracle[gpu-384-96]",
    "tests/test_ivf_pq_wide.py::test_wide_pq_edge_cases",
    "tests/test_ivf_pq_wide.py::test_wide_pq_reconstruct_matches_oracle",
]


def test_wide_pq_gpu_tests_on_the_emulated_library():
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


def _pair(d, nlist, M):
    from distributed_faiss_b200 import engine as E
    from oracle import oracle as O

    return E.GpuIndex(E.KIND_IVF_PQ, d, L2, nlist=nlist, pq_m=M), O.make_index("ivf_pq", d, metric=L2, nlist=nlist, M=M)


def _check_gpu_build(st, o, xb):
    """a shard trained and filled on the GPU: its codes and t-values are the oracle's encoding of
    the same rows with the same centroids and codebooks"""
    from oracle import oracle as O

    lists = O.assign(L2, st["centroids"], xb)
    order = np.argsort(lists, kind="stable")
    assert np.array_equal(st["ids"], order)
    enc = o._encode(xb[order], lists[order])
    assert st["codes"].tobytes() == enc["codes"].tobytes()
    assert st["tvals"].tobytes() == enc["tvals"].tobytes()


def _build_both(d, nlist, M, n, rs, via, niter=None):
    xb = clustered(rs, n, d, ncl=max(8, nlist // 2))
    g, o = _pair(d, nlist, M)
    if via == "gpu":
        if niter or EMU:
            g.set_param("kmeans_niter", niter or 2)
        g.train(xb[: n // 2])
        g.add(xb[: n // 3]); g.add(xb[n // 3:])
        st = g.get_state()
        o.set_state(st)
        _check_gpu_build(st, o, xb)
    else:
        o.train_niter = 4
        o.train(xb[: n // 2])
        o.add(xb)
        g.set_state(o.get_state())
        assert np.array_equal(g.get_array("tvals"), o.tvals)
    assert g.ntotal == n == o.ntotal
    return g, o, xb


@pytest.mark.gpu
@pytest.mark.parametrize("d,M", [(272, 68), (320, 80), (384, 96), (768, 128)])   # dsub 4, 4, 4, 6
@pytest.mark.parametrize("via", ["gpu", "oracle"])
def test_wide_pq_matches_oracle(d, M, via):
    rs = np.random.RandomState(10)
    nlist = 16
    g, o, xb = _build_both(d, nlist, M, _sz(6000, 1200), rs, via)
    xq = np.concatenate([clustered(rs, _sz(20, 4), d, ncl=8), xb[:3] + 0.01 * rs.randn(3, d).astype(np.float32)])
    for nprobe in (nlist, 1, 5):   # all lists; one; several probe groups per query
        g.nprobe = nprobe; o.nprobe = nprobe
        for k in ((1, 10, 33, 1024) if not EMU else (10, 1024)):   # 1024 > hits at nprobe 1: (FLT_MAX, -1) padding
            Dg, Ig = g.search(xq, k)
            Do, Io = o.search(xq, k)
            _assert_same(Dg, Ig, Do, Io, f"M={M} d={d} via={via} nprobe={nprobe} k={k}")
            assert g.last_stats()["ndis"] == o.last_ndis
        if nprobe == 1:
            assert (Ig == -1).any() and (Dg[Ig == -1] == FMAX).all()


@pytest.mark.gpu
def test_wide_pq_edge_cases():
    """k > hits, empty lists, nprobe > nlist, exact duplicate rows (ties broken by id)"""
    from oracle import oracle as O

    rs = np.random.RandomState(11)
    d, nlist, M = 160, 8, 80                                   # dsub 2
    xb = clustered(rs, 600, d, ncl=4, sigma=0.05)
    xb[10:20] = xb[0]
    o = O.make_index("ivf_pq", d, metric=L2, nlist=nlist, M=M)
    o.train_niter = 4
    o.train(xb); o.add(xb[:37])                                # few vectors: most lists empty
    g, _ = _pair(d, nlist, M)
    g.set_state(o.get_state())
    for nprobe in (1, 3, 50):
        g.nprobe = nprobe; o.nprobe = nprobe
        Dg, Ig = g.search(xb[:9], 64)
        Do, Io = o.search(xb[:9], 64)
        _assert_same(Dg, Ig, Do, Io, f"edge nprobe={nprobe}")
        assert (Ig == -1).any() and (Dg[Ig == -1] == FMAX).all()
        assert g.last_stats()["ndis"] == o.last_ndis
    row = Ig[0][Ig[0] >= 0].tolist()
    pos = [row.index(i) for i in [0] + list(range(10, 20))]
    assert pos == sorted(pos) and np.all(Dg[0][pos] == Dg[0][pos[0]])   # equal distances, ascending ids


@pytest.mark.gpu
def test_wide_pq_tensor_core_coarse_path_and_one_group_per_query():
    """nlist 1024 (tensor-core coarse quantizer at nprobe <= 512, FFMA at nprobe 1024), and a batch
    large enough that every query's probes go to one CTA"""
    if EMU:
        pytest.skip("too large for the emulator")
    rs = np.random.RandomState(12)
    d, nlist, M = 384, 1024, 96
    g, o, xb = _build_both(d, nlist, M, 40_000, rs, "gpu", niter=4)
    xq = np.concatenate([clustered(rs, 1200, d, ncl=64), xb[:8] + 0.01 * rs.randn(8, d).astype(np.float32)])
    for nprobe, nq in ((8, 1208), (1, 40), (16, 40), (1024, 8)):
        g.nprobe = nprobe; o.nprobe = nprobe
        for k in (10, 1024):
            Dg, Ig = g.search(xq[:nq], k)
            Do, Io = o.search(xq[:nq], k)
            _assert_same(Dg, Ig, Do, Io, f"nlist=1024 nprobe={nprobe} nq={nq} k={k}")
            assert g.last_stats()["ndis"] == o.last_ndis


@pytest.mark.gpu
def test_wide_pq_reconstruct_matches_oracle():
    rs = np.random.RandomState(14)
    g, o, xb = _build_both(384, 8, 96, _sz(3000, 800), rs, "oracle")
    ids = np.array([0, 5, len(xb) - 1, -1, 17], dtype=np.int64)
    R_g, R_o = g.reconstruct_rows(ids), o.reconstruct_rows(ids)
    assert np.isnan(R_g[3]).all()
    assert np.array_equal(R_g[[0, 1, 2, 4]], R_o[[0, 1, 2, 4]])
    g.nprobe = o.nprobe = 4
    Dg, Ig, Rg = g.search_and_reconstruct(xb[:6], 5)
    Do, Io, Ro = o.search_and_reconstruct(xb[:6], 5)
    _assert_same(Dg, Ig, Do, Io, "search_and_reconstruct")
    assert np.array_equal(Rg, Ro)


def _start_servers(n, root):
    import threading

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
def test_knnlm_code_size_96_sharded_through_the_client():
    """two IndexServers, knnlm with code_size=96: the client's merged answer is, bit for bit, the
    merge of what the oracle finds on each server's shard"""
    if EMU:
        pytest.skip("CUDA tensors")
    import tempfile

    from distributed_faiss_b200.index_cfg import IndexCfg
    from oracle import oracle as O
    from tests.test_gpu_api import make_client

    tmp = tempfile.TemporaryDirectory()
    servers, ports = _start_servers(2, tmp.name)
    try:
        rs = np.random.RandomState(16)
        d, nlist, M, k = 384, 8, 96, 20
        client = make_client(ports)
        cfg = IndexCfg(index_builder_type="knnlm", dim=d, centroids=nlist, metric="l2", train_num=1000, code_size=96)
        client.create_index("pq96", cfg)
        xs = [clustered(rs, 1000, d, ncl=8) for _ in range(4)]
        for b, x in enumerate(xs):
            client.add_index_data("pq96", x, list(range(1000 * b, 1000 * (b + 1))), False)
        client.sync_train("pq96")
        _wait_ntotal(client, "pq96", 4000)
        client.set_nprobe("pq96", 3)
        xq = np.concatenate(xs)[::211][:16] + np.float32(0.01)
        D, meta = client.search(xq, k, "pq96")
        Ds, Ps, metas = [], [], []
        for s in servers:
            ix = s.indexes["pq96"]
            assert ix.faiss_index.pq_m == M and ix.faiss_index.nprobe == 3
            o = O.make_index("ivf_pq", d, metric=L2, nlist=nlist, M=M)
            o.set_state(ix.faiss_index.get_state())
            o.nprobe = 3
            Do, Io = o.search(xq, k)
            Dg, Ig = ix.faiss_index.search(xq, k)
            _assert_same(Dg, Ig, Do, Io, f"shard {s}")
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


@pytest.mark.gpu
def test_factory_pq128_shard_saved_in_faiss_format_and_loaded_back():
    if EMU:
        pytest.skip("CUDA tensors")
    import tempfile

    from distributed_faiss_b200.index_cfg import IndexCfg
    from tests.test_gpu_api import make_client

    tmp = tempfile.TemporaryDirectory()
    servers, ports = _start_servers(1, tmp.name)
    try:
        rs = np.random.RandomState(17)
        d, index_id = 768, "pq128"
        cfg = IndexCfg(faiss_factory="IVF{centroids},PQ128", dim=d, centroids=8, metric="l2", train_num=1500,
                       index_format="faiss")
        client = make_client(ports)
        client.create_index(index_id, cfg)
        x = clustered(rs, 2000, d, ncl=8)
        client.add_index_data(index_id, x, list(range(2000)), False)
        client.sync_train(index_id)
        _wait_ntotal(client, index_id, 2000)
        client.set_nprobe(index_id, 4)
        D0, M0 = client.search(x[:9], 7, index_id)
        before = servers[0].indexes[index_id].faiss_index.get_state()
        assert before["M"] == 128 and before["codes"].shape == (2000, 128)
        client.save_index(index_id)
        assert os.path.isfile(os.path.join(tmp.name, index_id, "0", "index.faiss"))
        client.drop_index(index_id)
        client.close()
        c2 = make_client(ports)
        assert c2.load_index(index_id, cfg)
        c2.set_nprobe(index_id, 4)
        after = servers[0].indexes[index_id].faiss_index.get_state()
        for key in ("centroids", "codebooks", "list_off", "ids", "codes", "tvals"):
            assert np.asarray(after[key]).tobytes() == np.asarray(before[key]).tobytes(), key
        D1, M1 = c2.search(x[:9], 7, index_id)
        assert np.array_equal(D0, D1) and M0 == M1
        c2.close()
    finally:
        for s in servers:
            s.stop()
