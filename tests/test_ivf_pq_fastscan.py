"""IVF-PQ FastScan ("IVF{n},PQ{M}x4fs"): 4-bit codes of the raw vectors, searched through 8-bit
quantized distance tables and integer sums (dfx_scan_pq_fs_dev.cuh).

CPU: the factory parser, the oracle's invariants (table range, the dequantization bound against a
float64 restatement, flat tables, the ranking against float64 ADC), persistence, the faiss-format
refusal and sharded search through the servers with oracle engines; this file's `gpu` tests also run
against the emulated library.
GPU: the CUDA kernels against the oracle, bit for bit (distances, ids, ndis, codes, reconstruction), on
shards built on the GPU and imported from the oracle, the device-resident and graph-captured paths,
and the servers / client end to end."""
import os
import platform
import shutil
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


def _oracle_fs(d, nlist, M, n, rs, niter=4, ncl=None):
    from tests.oracle_pq_fs import OracleIVFPQFastScan

    o = OracleIVFPQFastScan(d, nlist, M)
    o.train_niter = niter
    xb = clustered(rs, n, d, ncl=ncl or max(4, nlist // 2))
    o.train(xb)
    o.add(xb)
    return o, xb


# ------------------------------------------------------------------ parser, CPU
@pytest.mark.parametrize("M", [8, 16, 32, 64, 128])
def test_parser_accepts_fastscan(M):
    from distributed_faiss_b200.factory import ACCEPTED_FORMS, FactorySpec, parse_factory

    assert "IVF{n},PQ{M}x4fs" in ACCEPTED_FORMS
    assert parse_factory(128, f"IVF4096,PQ{M}x4fs", L2) == FactorySpec("ivf_pq_fs", L2, 4096, M)


@pytest.mark.parametrize("s,d,match", [
    ("IVF64,PQ16x4fsr", 64, "not supported"),            # by_residual FastScan: per-list tables
    ("IVF64,PQ16x4fs_64", 64, "not supported"),          # block-size suffix
    ("IVF64,PQ16x4f", 64, "not supported"),
    ("IVF64,PQ16x4", 64, "not supported"),               # plain 4-bit PQ stays refused
    ("IVF64,PQ12x4fs", 96, "multiple of 8"),             # M % 8 != 0
    ("IVF64,PQ136x4fs", 272, "multiple of 8"),           # M > 128
    ("IVF64,PQ24x4fs", 64, "divides d=64"),              # M does not divide d
])
def test_parser_refuses_other_fastscan_forms(s, d, match):
    from distributed_faiss_b200.factory import ACCEPTED_FORMS, parse_factory

    with pytest.raises(RuntimeError, match=match) as e:
        parse_factory(d, s, L2)
    assert repr(s) in str(e.value)
    if match == "not supported":
        assert all(f in str(e.value) for f in ACCEPTED_FORMS)


def test_parser_refuses_inner_product_with_the_codec_message():
    from distributed_faiss_b200.factory import parse_factory
    from distributed_faiss_b200.index import factory_spec
    from distributed_faiss_b200.index_cfg import IndexCfg

    with pytest.raises(RuntimeError, match="inner-product distance tables"):
        parse_factory(64, "IVF64,PQ16x4fs", IP)
    with pytest.raises(RuntimeError, match="inner-product distance tables"):
        factory_spec(IndexCfg(faiss_factory="IVF{centroids},PQ16x4fs", dim=64, centroids=8, metric="dot"))
    # ivf_gpu: the raw string and faiss's default metric, L2, whatever cfg.metric says
    cfg = IndexCfg(index_builder_type="ivf_gpu", faiss_factory="IVF16,PQ8x4fs", dim=64, metric="dot", nprobe=3)
    assert factory_spec(cfg).kind == "ivf_pq_fs" and factory_spec(cfg).metric == L2


# ------------------------------------------------------------------ oracle invariants, CPU
def test_oracle_tables_stay_in_range_and_dequantize_within_the_bound(oracle_lib):
    from tests.oracle_pq_fs import adc_f64, dequant_bound, l2_tables, quantize_tables

    rs = np.random.RandomState(1)
    d, nlist, M = 64, 8, 16
    o, xb = _oracle_fs(d, nlist, M, 1500, rs)
    xq = np.concatenate([clustered(rs, 20, d, ncl=8), xb[:4] + np.float32(0.01), 3 * rs.randn(2, d).astype(np.float32)])
    lut = l2_tables(o.codebooks, xq)
    lutq, a, b, one_a = quantize_tables(lut)
    from tests.oracle_sq8 import fma32

    pre = np.floor(fma32((lut - lut.min(axis=2, keepdims=True)).astype(np.float32), a[:, None, None], np.float32(0.5)))
    assert pre.min() >= 0 and pre.max() <= 255 and np.array_equal(pre.astype(np.uint8), lutq)
    assert (lutq.min(axis=2) == 0).all()                      # every sub-table's minimum maps to 0
    assert (a > 0).all() and np.array_equal(one_a, (np.float32(1) / a).astype(np.float32))
    o.nprobe = 3
    D, I = o.search(xq, 50)
    st = o.get_state()
    inv = np.empty(o.ntotal, dtype=np.int64)
    inv[st["ids"]] = np.arange(o.ntotal)
    bound = dequant_bound(M, a)
    for q in range(len(xq)):
        ok = I[q] >= 0
        exact = adc_f64(st, xq[q:q + 1], inv[I[q][ok]])[0]
        slack = 1e-5 * (np.abs(exact) + 1)
        assert (np.abs(D[q][ok] - exact) <= bound[q] + slack).all(), q
    # reconstructions are the sub-centroids themselves (no coarse centroid is added)
    i0 = int(I[0][0])
    want = np.concatenate([st["codebooks"][m, st["codes"][inv[i0], m]] for m in range(M)])
    assert np.array_equal(o.reconstruct_rows(np.array([i0]))[0], want)


def test_oracle_flat_tables_pin_a_to_one(oracle_lib):
    from tests.oracle_pq_fs import quantize_tables

    lut = np.full((2, 8, 16), 3.25, dtype=np.float32)
    lut[1] = np.arange(8, dtype=np.float32)[:, None]          # flat sub-tables at different levels
    lutq, a, b, one_a = quantize_tables(lut)
    assert (a == 1).all() and (one_a == 1).all() and (lutq == 0).all()
    assert b[0] == np.float32(8 * 3.25) and b[1] == np.float32(28)


def test_oracle_ranking_is_float64_adc_where_the_gaps_exceed_the_bound(oracle_lib):
    from oracle import oracle as O
    from tests.oracle_pq_fs import adc_f64, dequant_bound, quantize_tables, l2_tables

    rs = np.random.RandomState(2)
    d, nlist, M, k = 64, 8, 8, 20
    o, xb = _oracle_fs(d, nlist, M, 2000, rs)
    o.nprobe = 4
    xq = np.concatenate([clustered(rs, 16, d, ncl=8), xb[:4] + np.float32(0.02)])
    D, I = o.search(xq, k)
    _, a, _, _ = quantize_tables(l2_tables(o.codebooks, xq))
    st = o.get_state()
    keys, _ = O.coarse(L2, st["centroids"], xq, 4)
    off = st["list_off"]
    for q in range(len(xq)):
        rows = np.concatenate([np.arange(off[l], off[l + 1]) for l in keys[q]]).astype(np.int64)
        adc = adc_f64(st, xq[q:q + 1], rows)[0]
        ids = st["ids"][rows]
        gap = 2 * (dequant_bound(M, a[q]) + 1e-5 * (np.abs(adc).max() + 1))
        kth = np.sort(adc)[k - 1]
        chosen = set(I[q].tolist())
        assert set(ids[adc < kth - gap].tolist()) <= chosen, q            # clearly in: returned
        assert all(v <= kth + gap for v in adc[np.isin(ids, I[q])]), q    # returned: never clearly out


# ------------------------------------------------------------------ persistence / servers, CPU
def _fs_cfg(d, M, **kw):
    from distributed_faiss_b200.index_cfg import IndexCfg

    return IndexCfg(faiss_factory=f"IVF{{centroids}},PQ{M}x4fs", dim=d, metric="l2", **kw)


def _wait_trained_index(ix):
    import time

    from distributed_faiss_b200.index_state import IndexState

    t0 = time.time()
    while ix.get_state() != IndexState.TRAINED:
        assert time.time() - t0 < 60, "index never reached TRAINED"
        time.sleep(0.01)


def test_fastscan_shard_saved_and_loaded_through_npz(oracle_lib, tmp_path):
    from distributed_faiss_b200 import faiss_io
    from distributed_faiss_b200.index import Index
    from distributed_faiss_b200.index_cfg import IndexCfg
    from tests.oracle_pq_fs import OracleIVFPQFastScan, oracle_engine_factory

    rs = np.random.RandomState(5)
    d, nlist, M = 32, 6, 16
    cfg = _fs_cfg(d, M, centroids=nlist, train_num=400, index_storage_dir=str(tmp_path))
    ix = Index(cfg, engine_factory=oracle_engine_factory)
    x = clustered(rs, 500, d, ncl=6)
    ix.add_batch(x, [("m", i) for i in range(500)], train_async_if_triggered=False)
    _wait_trained_index(ix)
    assert isinstance(ix.faiss_index, OracleIVFPQFastScan) and ix.faiss_index.nprobe == 1   # faiss default
    ix.set_nprobe(3)
    assert ix.save()
    q = x[::50] + np.float32(0.01)
    D1, m1, _ = ix.search(q, 7)
    cfg2 = IndexCfg.from_json(str(tmp_path / "cfg.json"))
    ix2 = Index.from_storage_dir(str(tmp_path), cfg2, engine_factory=oracle_engine_factory)
    ix2.set_nprobe(3)
    a, b = ix.faiss_index.get_state(), ix2.faiss_index.get_state()
    assert b["kind"] == "ivf_pq_fs" and "tvals" not in b
    for key in ("centroids", "codebooks", "list_off", "ids", "codes"):
        assert np.asarray(a[key]).tobytes() == np.asarray(b[key]).tobytes(), key
    D2, m2, _ = ix2.search(q, 7)
    assert D1.tobytes() == D2.tobytes() and m1 == m2
    # a cfg that builds another kind, or other (M, ksub), is refused (a cfg without a builder loads
    # with the stored one)
    def gpu_cfg(s):
        return IndexCfg(index_builder_type="ivf_gpu", faiss_factory=s, dim=d, metric="l2")

    with pytest.raises(RuntimeError, match="'ivf_pq_fs' but the cfg builds 'ivf_pq'"):
        Index.from_storage_dir(str(tmp_path), gpu_cfg(f"IVF{nlist},PQ{M}"), engine_factory=oracle_engine_factory)
    with pytest.raises(RuntimeError, match="'ivf_pq_fs' but the cfg builds 'ivf_pq'"):
        Index.from_storage_dir(str(tmp_path), IndexCfg(index_builder_type="knnlm", dim=d, centroids=nlist, metric="l2",
                                                       code_size=M, bits_per_vector=4),
                               engine_factory=oracle_engine_factory)
    with pytest.raises(RuntimeError, match=r"\(M, ksub\) = \(16, 16\) but the cfg builds \(8, 16\)"):
        Index.from_storage_dir(str(tmp_path), gpu_cfg(f"IVF{nlist},PQ8x4fs"), engine_factory=oracle_engine_factory)
    ix4 = Index.from_storage_dir(str(tmp_path), gpu_cfg(f"IVF{nlist},PQ{M}x4fs"), engine_factory=oracle_engine_factory)
    assert ix4.faiss_index.get_state()["codes"].tobytes() == a["codes"].tobytes()
    # the faiss format does not carry FastScan shards
    with pytest.raises(faiss_io.FaissFormatError, match="FastScan"):
        faiss_io.write_index(a, str(tmp_path / "x.faiss"))
    cfg3 = _fs_cfg(d, M, centroids=nlist, train_num=400, index_storage_dir=str(tmp_path / "f"), index_format="faiss")
    os.makedirs(cfg3.index_storage_dir)
    ix3 = Index(cfg3, engine_factory=oracle_engine_factory)
    ix3.add_batch(x, list(range(500)), train_async_if_triggered=False)
    _wait_trained_index(ix3)
    with pytest.raises(faiss_io.FaissFormatError, match="FastScan"):
        ix3.save()


def test_faiss_reader_refuses_fastscan_files(tmp_path):
    from distributed_faiss_b200 import faiss_io

    path = str(tmp_path / "pf.faiss")
    with open(path, "wb") as f:
        f.write(b"IwPf" + bytes(64))
    with pytest.raises(faiss_io.FaissFormatError, match="IwPf"):
        faiss_io.read_index(path)


def test_fastscan_sharded_search_is_the_merge_of_the_shards(oracle_lib):
    from distributed_faiss_b200.client import ResultHeap
    from distributed_faiss_b200.index_state import IndexState
    from distributed_faiss_b200.server import IndexServer
    from oracle import oracle as O
    from tests.oracle_engine import oracle_merge
    from tests.oracle_pq_fs import oracle_engine_factory
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
        client.create_index("fs", _fs_cfg(d, M, centroids=nlist, train_num=600))
        xs = [clustered(rs, 400, d, ncl=8) for _ in range(4)]
        for b, x in enumerate(xs):
            client.add_index_data("fs", x, list(range(400 * b, 400 * (b + 1))), False)
        client.sync_train("fs")
        wait_trained(client, "fs")
        import time

        t0 = time.time()
        while client.get_ntotal("fs") != 1600 or client.get_state("fs") != IndexState.TRAINED:
            assert time.time() - t0 < 60, "adds never finished"
            time.sleep(0.02)
        client.set_nprobe("fs", 3)
        xq = np.concatenate(xs)[::101][:12] + np.float32(0.01)
        D, meta = client.search(xq, k, "fs")
        Ds, Ps, metas = [], [], []
        for s in servers:
            ix = s.indexes["fs"]
            assert ix.faiss_index.kind == "ivf_pq_fs" and ix.faiss_index.M == M
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
    "tests/test_ivf_pq_fastscan.py::test_fs_matches_oracle[gpu-128-32]",
    "tests/test_ivf_pq_fastscan.py::test_fs_matches_oracle[oracle-96-24]",
    "tests/test_ivf_pq_fastscan.py::test_fs_matches_oracle[oracle-128-128]",
    "tests/test_ivf_pq_fastscan.py::test_fs_edge_cases",
    "tests/test_ivf_pq_fastscan.py::test_fs_reconstruct_matches_oracle",
    "tests/test_ivf_pq_fastscan.py::test_fs_limits",
]


def test_fs_gpu_tests_on_the_emulated_library():
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
    from tests.oracle_pq_fs import OracleIVFPQFastScan

    return (E.GpuIndex(E.KIND_IVF_PQ_FS, d, L2, nlist=nlist, pq_m=M, pq_nbits=4),
            OracleIVFPQFastScan(d, nlist, M))


def _build_both(d, nlist, M, n, rs, via, niter=None):
    from oracle import oracle as O
    from tests.oracle_pq_fs import encode

    xb = clustered(rs, n, d, ncl=max(8, nlist // 2))
    g, o = _pair(d, nlist, M)
    if via == "gpu":
        if niter or EMU:
            g.set_param("kmeans_niter", niter or 2)
        g.train(xb[: n // 2])
        g.add(xb[: n // 3]); g.add(xb[n // 3:])
        st = g.get_state()
        assert st["kind"] == "ivf_pq_fs" and st["ksub"] == 16 and st["codebooks"].shape == (M, 16, d // M)
        assert "tvals" not in st
        o.set_state(st)
        # device encoding: the oracle's codes of the same rows under the same centroids and codebooks
        lists = O.assign(L2, st["centroids"], xb)
        order = np.argsort(lists, kind="stable")
        assert np.array_equal(st["ids"], order)
        assert st["codes"].max() < 16 and st["codes"].tobytes() == encode(st["codebooks"], xb[order]).tobytes()
    else:
        o.train_niter = 4
        o.train(xb[: n // 2])
        o.add(xb)
        g.set_state(o.get_state())
        assert np.array_equal(g.get_array("codes").reshape(-1, M), o.codes)
    assert g.ntotal == n == o.ntotal
    return g, o, xb


@pytest.mark.gpu
@pytest.mark.parametrize("d,M", [(128, 8), (128, 16), (96, 24), (128, 32), (128, 64), (128, 128)])
@pytest.mark.parametrize("via", ["gpu", "oracle"])
def test_fs_matches_oracle(d, M, via):
    """distances, ids and ndis bit for bit, through the per-warp queues (k <= 1024) and the candidate
    rows (k > 1024)"""
    rs = np.random.RandomState(10)
    nlist = 16
    g, o, xb = _build_both(d, nlist, M, _sz(6000, 1200), rs, via)
    xq = np.concatenate([clustered(rs, _sz(20, 4), d, ncl=8), xb[:3] + 0.01 * rs.randn(3, d).astype(np.float32)])
    for nprobe in (nlist, 1, 5):   # all lists; one; several probe groups per query
        g.nprobe = nprobe; o.nprobe = nprobe
        for k in ((1, 10, 100, 1024, 1025, 4096) if not EMU else (10, 1025)):
            Dg, Ig = g.search(xq, k)
            Do, Io = o.search(xq, k)
            _assert_same(Dg, Ig, Do, Io, f"M={M} d={d} via={via} nprobe={nprobe} k={k}")
            assert g.last_stats()["ndis"] == o.last_ndis
        if nprobe == 1:
            assert (Ig == -1).any() and (Dg[Ig == -1] == FMAX).all()


@pytest.mark.gpu
def test_fs_edge_cases():
    """empty and single-vector lists, lists whose length is not a multiple of 32, exact duplicates
    (ties broken by id), k > hits, nprobe > nlist"""
    from tests.oracle_pq_fs import OracleIVFPQFastScan

    rs = np.random.RandomState(11)
    d, nlist, M = 64, 8, 16
    xb = clustered(rs, 600, d, ncl=4, sigma=0.05)
    xb[10:20] = xb[0]
    o = OracleIVFPQFastScan(d, nlist, M)
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
        for k in (1, 64, 1100):
            Dg, Ig = g.search(xq, k)
            Do, Io = o.search(xq, k)
            _assert_same(Dg, Ig, Do, Io, f"edge nprobe={nprobe} k={k}")
            assert g.last_stats()["ndis"] == o.last_ndis
        assert (Ig == -1).any() and (Dg[Ig == -1] == FMAX).all()
    Dg, Ig = g.search(xq, 64)
    assert Ig[-1][0] == 37                                        # the lone vector finds itself
    row = Ig[0][Ig[0] >= 0].tolist()
    pos = [row.index(i) for i in [0] + list(range(10, 20))]
    assert pos == sorted(pos) and np.all(Dg[0][pos] == Dg[0][pos[0]])   # equal distances, ascending ids


@pytest.mark.gpu
def test_fs_reconstruct_matches_oracle():
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
def test_fs_limits():
    from distributed_faiss_b200 import engine as E

    for M, d in ((8, 64), (24, 96), (128, 256)):
        E.GpuIndex(E.KIND_IVF_PQ_FS, d, L2, nlist=4, pq_m=M, pq_nbits=4)
    for M, d in ((4, 64), (12, 96), (136, 272), (20, 100)):
        with pytest.raises(RuntimeError, match=r"multiple of 8 in \[8, 128\] that divides d"):
            E.GpuIndex(E.KIND_IVF_PQ_FS, d, L2, nlist=4, pq_m=M, pq_nbits=4)
    for nbits in (8, 6):
        with pytest.raises(RuntimeError, match="4 bits per sub-quantizer"):
            E.GpuIndex(E.KIND_IVF_PQ_FS, 64, L2, nlist=4, pq_m=8, pq_nbits=nbits)
    with pytest.raises(RuntimeError, match="only the L2 metric"):
        E.GpuIndex(E.KIND_IVF_PQ_FS, 64, IP, nlist=4, pq_m=8, pq_nbits=4)
    # codes arrive one per byte and must fit in 4 bits
    rs = np.random.RandomState(16)
    o, _ = _oracle_fs(64, 4, 8, 200, rs)
    st = o.get_state()
    g, _ = _pair(64, 4, 8)
    bad = st["codes"].copy()
    bad[7, 3] = 16
    with pytest.raises(RuntimeError, match=r"4-bit code must be in \[0, 16\)"):
        g.set_state(dict(st, codes=bad))
    with pytest.raises(RuntimeError, match="no array named 'tvals'"):
        g.set_state(st)
        g.get_array("tvals")


@pytest.mark.gpu
def test_fs_many_queries_and_both_coarse_paths():
    """a batch of more queries than one chunk (k > 1024 chunks by the candidate rows), and the
    tensor-core coarse quantizer (nlist >= 1024) against the FFMA one"""
    if EMU:
        pytest.skip("too large for the emulator")
    rs = np.random.RandomState(12)
    d, nlist, M, n = 128, 16, 32, 6000
    g, o, xb = _build_both(d, nlist, M, n, rs, "oracle")
    g.nprobe = o.nprobe = nlist
    QC = (1 << 24) // n                   # one query's candidate row holds every vector
    xq = clustered(rs, QC + 300, d, ncl=8)
    Dg, Ig = g.search(xq, 1025)
    rows = np.array([0, 1, QC - 1, QC, QC + 1, len(xq) - 1])
    Do, Io = o.search(xq[rows], 1025)
    _assert_same(Dg[rows], Ig[rows], Do, Io, "chunk edges")
    D2, I2 = g.search(xq[QC - 2:QC + 2], 1025)
    _assert_same(Dg[QC - 2:QC + 2], Ig[QC - 2:QC + 2], D2, I2, "batch vs rows")

    rs = np.random.RandomState(13)
    g, o, xb = _build_both(128, 1024, 32, 20000, rs, "oracle")
    xq = np.concatenate([clustered(rs, 60, 128, ncl=8), xb[:4] + np.float32(0.01)])
    for nprobe in (1, 7):
        g.nprobe = o.nprobe = nprobe
        Do, Io = o.search(xq, 10)
        for tc in (1, 0):
            g.set_param("tensor_cores", tc)
            Dg, Ig = g.search(xq, 10)
            _assert_same(Dg, Ig, Do, Io, f"tensor_cores={tc} nprobe={nprobe}")
            assert g.last_stats()["ndis"] == o.last_ndis


@pytest.mark.gpu
def test_fs_device_paths_match_the_host_path(monkeypatch):
    """search_dev equals search; a ShardGroup of FastScan shards replays its search from a captured
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
        for k in (20, 1500):
            D, I = g.search(xq, k)
            Dd, Id = g.search_dev(x_t, k)
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
def test_fastscan_sharded_through_the_client_with_embeddings_and_npz_files():
    """two IndexServers on the GPU engine, an ivf_gpu "IVF8,PQ32x4fs" index: the client's merged answer
    (with return_embeddings) is the merge of the oracle's answers on each shard, and a save loads back
    into the same state and answers"""
    if EMU:
        pytest.skip("CUDA tensors")
    from distributed_faiss_b200.index_cfg import IndexCfg
    from oracle import oracle as O
    from tests.oracle_pq_fs import OracleIVFPQFastScan
    from tests.test_gpu_api import make_client

    tmp = tempfile.TemporaryDirectory()
    servers, ports = _start_servers(2, tmp.name)
    try:
        rs = np.random.RandomState(19)
        d, nlist, M, k, index_id = 128, 8, 32, 20, "fs"
        client = make_client(ports)
        # (metric="dot" would build the same L2 index, but the client would then rank the merge by -D)
        cfg = IndexCfg(index_builder_type="ivf_gpu", faiss_factory=f"IVF{nlist},PQ{M}x4fs", dim=d, metric="l2",
                       train_num=1000, nprobe=3)
        client.create_index(index_id, cfg)
        xs = [clustered(rs, 1000, d, ncl=8) for _ in range(4)]
        for b, x in enumerate(xs):
            client.add_index_data(index_id, x, list(range(1000 * b, 1000 * (b + 1))), False)
        client.sync_train(index_id)
        _wait_ntotal(client, index_id, 4000)
        xq = np.concatenate(xs)[::211][:16] + np.float32(0.01)
        D, meta, embs = client.search(xq, k, index_id, return_embeddings=True)
        Ds, Ps, Rs, metas, before = [], [], [], [], []
        for s in servers:
            ix = s.indexes[index_id]
            assert ix.faiss_index.kind == 5 and ix.faiss_index.nprobe == 3 and ix.faiss_index.metric == L2
            st = ix.faiss_index.get_state()
            before.append(st)
            o = OracleIVFPQFastScan(d, nlist, M)
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
        assert os.path.isfile(os.path.join(tmp.name, index_id, "0", "index.dfx.npz"))
        client.drop_index(index_id)
        client.close()
        c2 = make_client(ports)
        assert c2.load_index(index_id, cfg)
        for s, st in zip(servers, before):
            after = s.indexes[index_id].faiss_index.get_state()
            for key in ("centroids", "codebooks", "list_off", "ids", "codes"):
                assert np.asarray(after[key]).tobytes() == np.asarray(st[key]).tobytes(), key
        D1, M1 = c2.search(xq, k, index_id)
        assert np.array_equal(np.asarray(D1, dtype=np.float32), refD) and M1 == meta
        c2.close()
    finally:
        for s in servers:
            s.stop()
