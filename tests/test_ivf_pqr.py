"""IVF-PQR ("IVF{n},PQ{M}+{M2}"): IVF-PQ candidates re-ranked on a second, M2-byte residual code
(dfx_refine_dev.cuh).

CPU: the factory parser, the oracle against a float64 restatement, the recall gain the refinement
exists for, persistence (npz and the faiss format "IwQR") and sharded search through the servers with
oracle engines; this file's `gpu` tests also run against the emulated library.
GPU: the CUDA kernels against the oracle, bit for bit (distances, ids, ndis, codes, refine codes,
reconstruction), on shards built on the GPU and imported from the oracle, the device-resident and
graph-captured paths, and the servers / client end to end."""
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


def _oracle_pqr(d, nlist, M, M2, n, rs, niter=4, ncl=None):
    from tests.oracle_pqr import OracleIVFPQR

    o = OracleIVFPQR(d, nlist, M, M2)
    o.train_niter = niter
    xb = clustered(rs, n, d, ncl=ncl or max(4, nlist // 2))
    o.train(xb)
    o.add(xb)
    return o, xb


# ------------------------------------------------------------------ parser, CPU
@pytest.mark.parametrize("M,M2", [(4, 4), (8, 16), (16, 16), (32, 8), (64, 128), (128, 32)])
def test_parser_accepts_pqr(M, M2):
    from distributed_faiss_b200.factory import ACCEPTED_FORMS, FactorySpec, parse_factory

    assert "IVF{n},PQ{M}+{M2}" in ACCEPTED_FORMS
    spec = parse_factory(128, f"IVF4096,PQ{M}+{M2}", L2)
    assert spec == FactorySpec("ivf_pqr", L2, 4096, M, M2) and spec.refine_m == M2
    assert parse_factory(128, f"IVF4096,PQ{M}", L2).refine_m == 0   # the other kinds keep refine_m = 0


@pytest.mark.parametrize("s,d,match", [
    ("IVF64,PQ16+24", 64, "divides d=64"),                # M2 does not divide d
    ("IVF64,PQ16+6", 96, "multiple of 4"),                # M2 % 4 != 0
    ("IVF64,PQ16+136", 272, "at most 128"),               # M2 > 128
    ("IVF64,PQ12+16", 64, "divides d=64"),                # M does not divide d
    ("IVF64,PQ16+0", 64, "not supported"),
    ("IVF64,PQ16x8+16", 64, "not supported"),
    ("IVF64,PQ16+16x8", 64, "not supported"),
    ("IVF64,PQ16x4fs+16", 64, "not supported"),
    ("IVF64,PQ16+", 64, "not supported"),
])
def test_parser_refuses_other_pqr_forms(s, d, match):
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
        parse_factory(64, "IVF64,PQ16+16", IP)
    with pytest.raises(RuntimeError, match="inner-product distance tables"):
        factory_spec(IndexCfg(faiss_factory="IVF{centroids},PQ16+8", dim=64, centroids=8, metric="dot"))
    # ivf_gpu: the raw string and faiss's default metric, L2, whatever cfg.metric says
    cfg = IndexCfg(index_builder_type="ivf_gpu", faiss_factory="IVF16,PQ8+16", dim=64, metric="dot", nprobe=3)
    spec = factory_spec(cfg)
    assert spec.kind == "ivf_pqr" and spec.metric == L2 and (spec.pq_m, spec.refine_m) == (8, 16)


# ------------------------------------------------------------------ oracle, CPU
def test_first_stage_k_is_the_fp32_product():
    from tests.oracle_pqr import first_stage_k

    assert first_stage_k(10, 4.0) == 40 and first_stage_k(1025, 2.5) == 2562 and first_stage_k(4096, 4) == 16384
    assert first_stage_k(3, 1.0) == 3 and first_stage_k(7, 1.3) == int(np.float32(7) * np.float32(1.3))


def test_oracle_warp_l2_is_oracle_warp_dot(oracle_lib):
    from oracle import oracle as O
    from tests.oracle_pqr import warp_l2

    rs = np.random.RandomState(0)
    for d in (4, 60, 128, 196, 256):
        a = rs.randn(5, d).astype(np.float32)
        got = warp_l2(a)
        want = [O.warp_dot(a[i], np.zeros(d, np.float32), 1) for i in range(5)]
        assert np.array_equal(got, np.array(want, dtype=np.float32)), d


def test_oracle_matches_a_float64_restatement(oracle_lib):
    """distances within fp32 rounding of float64 |q - ((c + p1) + p2)|^2, and the ids are those of
    float64 wherever its distances are separated by more than that rounding"""
    from oracle import oracle as O
    from tests.oracle_pqr import reconstruct_f64

    rs = np.random.RandomState(1)
    d, nlist, M, M2, k = 64, 8, 8, 16, 10
    o, xb = _oracle_pqr(d, nlist, M, M2, 2000, rs)
    o.nprobe = 3
    xq = np.concatenate([clustered(rs, 16, d, ncl=8), xb[:4] + np.float32(0.01)])
    D, I = o.search(xq, k)
    _, I1 = O.OracleIVFPQ.search(o, xq, 4 * k)   # the first stage's candidates
    st = o.get_state()
    inv = np.empty(o.ntotal, dtype=np.int64)
    inv[st["ids"]] = np.arange(o.ntotal)
    for q in range(len(xq)):
        cand = I1[q][I1[q] >= 0]
        exact = ((xq[q].astype(np.float64) - reconstruct_f64(st, inv[cand])) ** 2).sum(axis=1)
        tol = 1e-5 * (exact.max() + (xq[q].astype(np.float64) ** 2).sum() + 1)
        got = dict(zip(I[q].tolist(), D[q].tolist()))
        for i, e in zip(cand.tolist(), exact.tolist()):
            if i in got:
                assert abs(got[i] - e) <= tol, (q, i)
        kth = np.sort(exact)[k - 1]
        assert set(cand[exact < kth - 2 * tol].tolist()) <= set(I[q].tolist()), q   # clearly in: returned
        assert all(e <= kth + 2 * tol for i, e in zip(cand.tolist(), exact.tolist()) if i in got), q
    # reconstruction: (c + p1) + p2 in fp32
    i0 = int(I[0][0])
    pos = inv[i0]
    lo = o.list_of_rows()[pos]
    p1 = np.concatenate([st["codebooks"][m, st["codes"][pos, m]] for m in range(M)])
    p2 = np.concatenate([st["refine_codebooks"][m, st["refine_codes"][i0, m]] for m in range(M2)])
    assert np.array_equal(o.reconstruct_rows(np.array([i0]))[0], (st["centroids"][lo] + p1) + p2)


def _recall(I, gt):
    return np.mean([len(set(a.tolist()) & set(b.tolist())) / gt.shape[1] for a, b in zip(I, gt)])


def test_refinement_raises_recall_on_clustered_data(oracle_lib):
    """the point of the kind: on seeded clustered data PQ{M}+{M2} has a higher mean recall@10 than
    PQ{M} over the same lists and codes"""
    from oracle import oracle as O

    rs = np.random.RandomState(2)
    d, nlist, M, M2, k = 64, 16, 8, 8, 10
    o, xb = _oracle_pqr(d, nlist, M, M2, 4000, rs, ncl=64)
    o.nprobe = 4
    xq = clustered(np.random.RandomState(3), 100, d, ncl=64)
    _, gt = O.flat_search(L2, xb, xq, k)
    _, I_pq = O.OracleIVFPQ.search(o, xq, k)
    _, I_pqr = o.search(xq, k)
    r_pq, r_pqr = _recall(I_pq, gt), _recall(I_pqr, gt)
    assert r_pqr > r_pq + 0.05, (r_pq, r_pqr)


# ------------------------------------------------------------------ persistence / servers, CPU
def _pqr_cfg(d, M, M2, **kw):
    from distributed_faiss_b200.index_cfg import IndexCfg

    return IndexCfg(faiss_factory=f"IVF{{centroids}},PQ{M}+{M2}", dim=d, metric="l2", **kw)


def _wait_trained_index(ix):
    import time

    from distributed_faiss_b200.index_state import IndexState

    t0 = time.time()
    while ix.get_state() != IndexState.TRAINED:
        assert time.time() - t0 < 60, "index never reached TRAINED"
        time.sleep(0.01)


STATE_KEYS = ("centroids", "codebooks", "list_off", "ids", "codes", "refine_codebooks", "refine_codes")


def test_iwqr_round_trip(oracle_lib, tmp_path):
    from distributed_faiss_b200 import faiss_io

    rs = np.random.RandomState(4)
    o, _ = _oracle_pqr(32, 6, 8, 16, 500, rs)
    o.k_factor = 2.5
    st = o.get_state()
    path = str(tmp_path / "pqr.faiss")
    faiss_io.write_index(st, path, nprobe=3)
    with open(path, "rb") as f:
        assert f.read(4) == b"IwQR"
    back, nprobe = faiss_io.read_index(path)
    assert nprobe == 3 and back["kind"] == "ivf_pqr" and back["M2"] == 16 and back["k_factor"] == 2.5
    for key in STATE_KEYS:
        assert np.asarray(back[key]).tobytes() == np.asarray(st[key]).tobytes(), key
    # an IwPQ file is read as plain IVF-PQ, exactly as before
    plain = {k: v for k, v in st.items() if k not in ("M2", "refine_codebooks", "refine_codes", "k_factor")}
    faiss_io.write_index(dict(plain, kind="ivf_pq"), str(tmp_path / "pq.faiss"))
    back_pq, _ = faiss_io.read_index(str(tmp_path / "pq.faiss"))
    assert back_pq["kind"] == "ivf_pq" and "M2" not in back_pq
    # a refine-code block that does not hold ntotal rows is refused
    raw = open(path, "rb").read()
    with open(str(tmp_path / "cut.faiss"), "wb") as f:
        f.write(raw[:-4 - 16 * 3])
    with pytest.raises(faiss_io.FaissFormatError):
        faiss_io.read_index(str(tmp_path / "cut.faiss"))


def test_pqr_shard_saved_and_loaded_through_npz_and_faiss(oracle_lib, tmp_path):
    from distributed_faiss_b200.index import Index
    from distributed_faiss_b200.index_cfg import IndexCfg
    from tests.oracle_pqr import OracleIVFPQR, oracle_engine_factory

    rs = np.random.RandomState(5)
    d, nlist, M, M2 = 32, 6, 8, 16
    x = clustered(rs, 500, d, ncl=6)
    q = x[::50] + np.float32(0.01)
    for fmt in ("dfx", "faiss"):
        root = tmp_path / fmt
        os.makedirs(root)
        cfg = _pqr_cfg(d, M, M2, centroids=nlist, train_num=400, index_storage_dir=str(root), index_format=fmt)
        ix = Index(cfg, engine_factory=oracle_engine_factory)
        ix.add_batch(x, [("m", i) for i in range(500)], train_async_if_triggered=False)
        _wait_trained_index(ix)
        assert isinstance(ix.faiss_index, OracleIVFPQR) and ix.faiss_index.nprobe == 1   # faiss default
        ix.faiss_index.k_factor = 3.0
        ix.set_nprobe(3)
        assert ix.save()
        D1, m1, _ = ix.search(q, 7)
        cfg2 = IndexCfg.from_json(str(root / "cfg.json"))
        ix2 = Index.from_storage_dir(str(root), cfg2, engine_factory=oracle_engine_factory)
        ix2.set_nprobe(3)
        a, b = ix.faiss_index.get_state(), ix2.faiss_index.get_state()
        assert b["kind"] == "ivf_pqr" and b["k_factor"] == 3.0
        for key in STATE_KEYS:
            assert np.asarray(a[key]).tobytes() == np.asarray(b[key]).tobytes(), (fmt, key)
        D2, m2, _ = ix2.search(q, 7)
        assert D1.tobytes() == D2.tobytes() and m1 == m2

    def gpu_cfg(s):
        return IndexCfg(index_builder_type="ivf_gpu", faiss_factory=s, dim=d, metric="l2")

    root = str(tmp_path / "dfx")
    with pytest.raises(RuntimeError, match=r"\(M, ksub, M2\) = \(8, 256, 16\) but the cfg builds \(8, 256, 8\)"):
        Index.from_storage_dir(root, gpu_cfg(f"IVF{nlist},PQ{M}+8"), engine_factory=oracle_engine_factory)
    with pytest.raises(RuntimeError, match=r"\(M, ksub, M2\) = \(8, 256, 16\) but the cfg builds \(16, 256, 16\)"):
        Index.from_storage_dir(root, gpu_cfg(f"IVF{nlist},PQ16+{M2}"), engine_factory=oracle_engine_factory)
    with pytest.raises(RuntimeError, match="'ivf_pqr' but the cfg builds 'ivf_pq'"):
        Index.from_storage_dir(root, gpu_cfg(f"IVF{nlist},PQ{M}"), engine_factory=oracle_engine_factory)
    ix4 = Index.from_storage_dir(root, gpu_cfg(f"IVF{nlist},PQ{M}+{M2}"), engine_factory=oracle_engine_factory)
    assert ix4.faiss_index.get_state()["refine_codes"].shape == (500, M2)


def test_pqr_sharded_search_is_the_merge_of_the_shards(oracle_lib):
    from distributed_faiss_b200.client import ResultHeap
    from distributed_faiss_b200.index_state import IndexState
    from distributed_faiss_b200.server import IndexServer
    from oracle import oracle as O
    from tests.oracle_engine import oracle_merge
    from tests.oracle_pqr import oracle_engine_factory
    from tests.test_host_logic import free_ports, make_client, wait_listening, wait_trained

    ResultHeap.merge_backend = staticmethod(oracle_merge)
    tmp = tempfile.TemporaryDirectory()
    ports = free_ports(3)
    servers = [IndexServer(r, tmp.name, engine_factory=oracle_engine_factory) for r in range(3)]
    for s, p in zip(servers, ports):
        threading.Thread(target=s.start_blocking, args=(p,), daemon=True).start()
    wait_listening(ports)
    try:
        rs = np.random.RandomState(6)
        d, nlist, M, M2, k = 64, 8, 16, 8, 12
        client = make_client(ports)
        client.create_index("pqr", _pqr_cfg(d, M, M2, centroids=nlist, train_num=600))
        xs = [clustered(rs, 400, d, ncl=8) for _ in range(6)]
        for b, x in enumerate(xs):
            client.add_index_data("pqr", x, list(range(400 * b, 400 * (b + 1))), False)
        client.sync_train("pqr")
        wait_trained(client, "pqr")
        import time

        t0 = time.time()
        while client.get_ntotal("pqr") != 2400 or client.get_state("pqr") != IndexState.TRAINED:
            assert time.time() - t0 < 60, "adds never finished"
            time.sleep(0.02)
        client.set_nprobe("pqr", 3)
        xq = np.concatenate(xs)[::101][:12] + np.float32(0.01)
        D, meta = client.search(xq, k, "pqr")
        Ds, Ps, metas = [], [], []
        for s in servers:
            ix = s.indexes["pqr"]
            assert ix.faiss_index.kind == "ivf_pqr" and ix.faiss_index.M2 == M2
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
    "tests/test_ivf_pqr.py::test_pqr_matches_oracle[gpu-128-32-16-1]",
    "tests/test_ivf_pqr.py::test_pqr_matches_oracle[oracle-128-32-8-0]",
    "tests/test_ivf_pqr.py::test_pqr_matches_oracle[oracle-96-48-24-1]",
    "tests/test_ivf_pqr.py::test_pqr_edge_cases",
    "tests/test_ivf_pqr.py::test_pqr_reconstruct_matches_oracle",
    "tests/test_ivf_pqr.py::test_pqr_limits",
]


def test_pqr_gpu_tests_on_the_emulated_library():
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


def _pair(d, nlist, M, M2):
    from distributed_faiss_b200 import engine as E
    from tests.oracle_pqr import OracleIVFPQR

    return (E.GpuIndex(E.KIND_IVF_PQR, d, L2, nlist=nlist, pq_m=M, pq_nbits=8, refine_m=M2),
            OracleIVFPQR(d, nlist, M, M2))


def _build_both(d, nlist, M, M2, n, rs, via, niter=None, il=1):
    from oracle import oracle as O
    from tests.oracle_pqr import encode

    xb = clustered(rs, n, d, ncl=max(8, nlist // 2))
    g, o = _pair(d, nlist, M, M2)
    g.set_param("interleaved", il)
    if via == "gpu":
        if niter or EMU:
            g.set_param("kmeans_niter", niter or 2)
        g.train(xb[: n // 2])
        g.add(xb[: n // 3]); g.add(xb[n // 3:])
        st = g.get_state()
        assert st["kind"] == "ivf_pqr" and st["ksub"] == 256 and st["M2"] == M2
        assert st["refine_codebooks"].shape == (M2, 256, d // M2) and st["k_factor"] == 4.0
        o.set_state(st)
        # device encoding: the oracle's codes and refine codes of the same rows under the same centroids
        # and codebooks; ids in the stable list order
        lists = O.assign(L2, st["centroids"], xb)
        order = np.argsort(lists, kind="stable")
        assert np.array_equal(st["ids"], order)
        codes = O.OracleIVFPQ._encode(o, xb, lists)["codes"]
        assert st["codes"].tobytes() == codes[order].tobytes()
        assert st["refine_codes"].tobytes() == encode(st["refine_codebooks"], o.residual2(xb, lists, codes)).tobytes()
    else:
        o.train_niter = 4
        o.train(xb[: n // 2])
        o.add(xb)
        g.set_state(o.get_state())
        assert np.array_equal(g.get_array("codes").reshape(-1, M), o.codes)
        assert np.array_equal(g.get_array("refine_codes").reshape(-1, M2), o.refine_codes)
    assert g.ntotal == n == o.ntotal
    return g, o, xb


@pytest.mark.gpu
@pytest.mark.parametrize("d,M,M2,il", [(128, 8, 16, 1), (128, 16, 16, 1), (128, 32, 16, 1), (128, 32, 8, 0),
                                       (96, 48, 24, 1), (128, 64, 32, 1), (192, 96, 48, 1), (128, 128, 64, 1)])
@pytest.mark.parametrize("via", ["gpu", "oracle"])
def test_pqr_matches_oracle(d, M, M2, il, via):
    """distances, ids and ndis bit for bit; k' = 4k crosses 1024 (candidate rows) and 4096 and reaches
    16384 at k = 4096.  M = 32 covers the interleaved scan (il = 1) and the row-major one (il = 0)"""
    rs = np.random.RandomState(10)
    nlist = 16
    g, o, xb = _build_both(d, nlist, M, M2, _sz(6000, 1200), rs, via, il=il)
    assert g.get_param("interleaved") == il
    xq = np.concatenate([clustered(rs, _sz(12, 4), d, ncl=8), xb[:3] + 0.01 * rs.randn(3, d).astype(np.float32)])
    for nprobe in (nlist, 1, 5):   # all lists; one; several probe groups per query
        g.nprobe = nprobe; o.nprobe = nprobe
        for k in ((1, 10, 100, 1024, 1025, 4096) if not EMU else (10, 300)):
            Dg, Ig = g.search(xq, k)
            Do, Io = o.search(xq, k)
            _assert_same(Dg, Ig, Do, Io, f"M={M} M2={M2} d={d} via={via} nprobe={nprobe} k={k}")
            assert g.last_stats()["ndis"] == o.last_ndis
        if nprobe == 1:
            assert (Ig == -1).any() and (Dg[Ig == -1] == FMAX).all()


@pytest.mark.gpu
@pytest.mark.parametrize("k_factor", [1, 2.5, 4])
def test_pqr_k_factor(k_factor):
    rs = np.random.RandomState(15)
    g, o, xb = _build_both(128, 16, 16, 32, _sz(5000, 1000), rs, "oracle")
    g.set_param("k_factor", k_factor)
    o.k_factor = k_factor
    assert g.get_param("k_factor") == k_factor and g.get_state()["k_factor"] == k_factor
    xq = np.concatenate([clustered(rs, _sz(20, 4), 128, ncl=8), xb[:3] + np.float32(0.01)])
    for nprobe in (1, 6):
        g.nprobe = o.nprobe = nprobe
        for k in (1, 7, 100, 1025, 4096):
            Dg, Ig = g.search(xq, k)
            Do, Io = o.search(xq, k)
            _assert_same(Dg, Ig, Do, Io, f"k_factor={k_factor} nprobe={nprobe} k={k}")


@pytest.mark.gpu
def test_pqr_edge_cases():
    """empty and single-vector lists, fewer than k' vectors probed, exact duplicates (ties broken by id),
    k > hits, nprobe > nlist"""
    from tests.oracle_pqr import OracleIVFPQR

    rs = np.random.RandomState(11)
    d, nlist, M, M2 = 64, 8, 16, 8
    xb = clustered(rs, 600, d, ncl=4, sigma=0.05)
    xb[10:20] = xb[0]
    o = OracleIVFPQR(d, nlist, M, M2)
    o.train_niter = 4
    o.train(xb)
    far = (100.0 + rs.randn(1, d)).astype(np.float32)
    o.centroids[-1] = far[0]                                    # the last list holds `far` alone
    o.add(np.concatenate([xb[:37], far]))
    sizes = np.diff(o.list_off)
    assert sizes[-1] == 1 and (sizes == 0).any() and (sizes % 32 != 0).any()
    for il in (1, 0):
        g, _ = _pair(d, nlist, M, M2)
        g.set_param("interleaved", il)
        g.set_state(o.get_state())
        xq = np.concatenate([xb[:9], far])
        for nprobe in (1, 3, 50):
            g.nprobe = nprobe; o.nprobe = nprobe
            for k in (1, 5, 64, 1100):
                Dg, Ig = g.search(xq, k)
                Do, Io = o.search(xq, k)
                _assert_same(Dg, Ig, Do, Io, f"edge il={il} nprobe={nprobe} k={k}")
                assert g.last_stats()["ndis"] == o.last_ndis
            assert (Ig == -1).any() and (Dg[Ig == -1] == FMAX).all()
        Dg, Ig = g.search(xq, 64)
        assert Ig[-1][0] == 37                                        # the lone vector finds itself
        row = Ig[0][Ig[0] >= 0].tolist()
        pos = [row.index(i) for i in [0] + list(range(10, 20))]
        assert pos == sorted(pos) and np.all(Dg[0][pos] == Dg[0][pos[0]])   # equal distances, ascending ids
    # an empty trained index answers with padding only
    g, _ = _pair(d, nlist, M, M2)
    g.set_param("kmeans_niter", 2)
    g.train(xb)
    D, I = g.search(xb[:3], 5)
    assert (I == -1).all() and (D == FMAX).all()


@pytest.mark.gpu
def test_pqr_reconstruct_matches_oracle():
    rs = np.random.RandomState(14)
    for il in (1, 0):
        g, o, xb = _build_both(128, 8, 32, 16, _sz(3000, 800), rs, "oracle", il=il)
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
def test_pqr_limits():
    from distributed_faiss_b200 import engine as E

    for M, M2, d in ((4, 4, 64), (128, 128, 256), (8, 64, 64)):
        E.GpuIndex(E.KIND_IVF_PQR, d, L2, nlist=4, pq_m=M, refine_m=M2)
    for M2, d in ((0, 64), (6, 96), (136, 272), (24, 100), (12, 64)):
        with pytest.raises(RuntimeError, match="refinement sub-quantizers must be a multiple of 4"):
            E.GpuIndex(E.KIND_IVF_PQR, d, L2, nlist=4, pq_m=4, refine_m=M2)
    with pytest.raises(RuntimeError, match="IVF-PQR: the number of sub-quantizers"):
        E.GpuIndex(E.KIND_IVF_PQR, 64, L2, nlist=4, pq_m=12, refine_m=8)
    with pytest.raises(RuntimeError, match="8 bits per sub-quantizer"):
        E.GpuIndex(E.KIND_IVF_PQR, 64, L2, nlist=4, pq_m=8, pq_nbits=4, refine_m=8)
    with pytest.raises(RuntimeError, match="only the L2 metric"):
        E.GpuIndex(E.KIND_IVF_PQR, 64, IP, nlist=4, pq_m=8, refine_m=8)
    with pytest.raises(RuntimeError, match="refine_m must be 0"):
        E.GpuIndex(E.KIND_IVF_PQ, 64, L2, nlist=4, pq_m=8, refine_m=8)
    rs = np.random.RandomState(16)
    o, _ = _oracle_pqr(64, 4, 8, 8, 300, rs)
    st = o.get_state()
    g, _ = _pair(64, 4, 8, 8)
    # k_factor below 1 is refused; a k' beyond 16384 raises before anything is launched
    for bad in (0.5, 0, -1):
        with pytest.raises(RuntimeError, match=r"k_factor must be in \[1, 16384\]"):
            g.set_param("k_factor", bad)
    with pytest.raises(RuntimeError, match="k_factor is a parameter of IVF-PQR"):
        E.GpuIndex(E.KIND_IVF_PQ, 64, L2, nlist=4, pq_m=8).set_param("k_factor", 2)
    g.set_state(st)
    g.set_param("k_factor", 4.5)
    n0 = E.launch_count()
    with pytest.raises(RuntimeError, match=r"k=4096 with k_factor=4\.5.*18432 candidates to re-rank, more than 16384"):
        g.search(st["centroids"][:2], 4096)
    with pytest.raises(RuntimeError, match="IVF search supports k <= 4096"):
        g.search(st["centroids"][:2], 4097)
    assert E.launch_count() == n0
    g.set_param("k_factor", 4)
    D, I = g.search(st["centroids"][:2], 4096)
    assert (I[:, 300:] == -1).all()
    # the ids of an import must be a permutation of 0 .. ntotal-1: the refine codes are addressed by id
    bad = st["ids"].copy()
    bad[[3, 4]] = bad[3]
    g2, _ = _pair(64, 4, 8, 8)
    with pytest.raises(RuntimeError, match="permutation"):
        g2.set_state(dict(st, ids=bad))
    with pytest.raises(RuntimeError, match="refine_codes: wrong size"):
        g2.set_state(dict(st, refine_codes=st["refine_codes"][:-1]))
    with pytest.raises(RuntimeError, match="refine_codebooks: wrong size"):
        g2.set_array("refine_codebooks", st["refine_codebooks"].reshape(-1)[:-1])
    from tests.test_gpu_parity import _import_without

    for skip, msg in (("refine_codebooks", "refine_codebooks are required"),
                      ("refine_codes", "refine_codes of every vector are required")):
        with pytest.raises(RuntimeError, match="import: " + msg):
            _import_without(_pair(64, 4, 8, 8)[0], st, skip)


@pytest.mark.gpu
def test_pqr_many_queries_and_both_coarse_paths():
    """a batch of more queries than one chunk (the re-ranking chunks by k', the candidate rows by the
    lists), and the tensor-core coarse quantizer (nlist >= 1024) against the FFMA one"""
    if EMU:
        pytest.skip("too large for the emulator")
    rs = np.random.RandomState(12)
    d, nlist, M, M2, n = 128, 16, 32, 16, 6000
    g, o, xb = _build_both(d, nlist, M, M2, n, rs, "oracle")
    g.nprobe = o.nprobe = nlist
    QC = (1 << 22) // 4100                # the re-ranking chunk at k' = 4 * 1025
    xq = clustered(rs, QC + 300, d, ncl=8)
    Dg, Ig = g.search(xq, 1025)
    rows = np.array([0, 1, QC - 1, QC, QC + 1, len(xq) - 1])
    Do, Io = o.search(xq[rows], 1025)
    _assert_same(Dg[rows], Ig[rows], Do, Io, "chunk edges")
    D2, I2 = g.search(xq[QC - 2:QC + 2], 1025)
    _assert_same(Dg[QC - 2:QC + 2], Ig[QC - 2:QC + 2], D2, I2, "batch vs rows")
    Dg, Ig = g.search(xq, 10)             # k' = 40: the per-warp queues, 8192-query chunks
    Do, Io = o.search(xq[rows], 10)
    _assert_same(Dg[rows], Ig[rows], Do, Io, "k=10 batch")

    rs = np.random.RandomState(13)
    g, o, xb = _build_both(128, 1024, 32, 32, 20000, rs, "oracle")
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
def test_pqr_refine_stage_is_timed_on_its_own():
    if EMU:
        pytest.skip("CUDA events")
    rs = np.random.RandomState(18)
    g, o, xb = _build_both(128, 16, 16, 16, 4000, rs, "oracle")
    g.nprobe = 4
    g.profile(True)
    g.search(xb[:100], 10)
    g.search(xb[:100], 10)
    assert g.get_param("refine_launches") == 2 and g.get_param("refine_ms") > 0
    scan_ms, scans = g.profile_read(reset=True)
    assert scans == 2 and scan_ms > 0
    assert g.get_param("refine_launches") == 0
    g.profile(False)


@pytest.mark.gpu
def test_pqr_device_paths_match_the_host_path(monkeypatch):
    """search_dev equals search; a ShardGroup of IVF-PQR shards replays its search from a captured
    CUDA graph with the eager answers"""
    if EMU:
        pytest.skip("CUDA tensors")
    import torch

    from distributed_faiss_b200 import spmd

    rs = np.random.RandomState(17)
    shards, tables, base = [], [], 0
    for s in range(2):
        g, o, xb = _build_both(128, 32, 32 if s == 0 else 16, 16, 8000, rs, "gpu")
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
def test_pqr_sharded_through_the_client_with_embeddings_and_saved_files():
    """two IndexServers on the GPU engine, an ivf_gpu "IVF8,PQ16+16" index: the client's merged answer
    (with return_embeddings) is the merge of the oracle's answers on each shard, and a save in the
    faiss format loads back into the same state and answers"""
    if EMU:
        pytest.skip("CUDA tensors")
    from distributed_faiss_b200.index_cfg import IndexCfg
    from oracle import oracle as O
    from tests.oracle_pqr import OracleIVFPQR
    from tests.test_gpu_api import make_client

    tmp = tempfile.TemporaryDirectory()
    servers, ports = _start_servers(2, tmp.name)
    try:
        rs = np.random.RandomState(19)
        d, nlist, M, M2, k, index_id = 128, 8, 16, 16, 20, "pqr"
        client = make_client(ports)
        cfg = IndexCfg(index_builder_type="ivf_gpu", faiss_factory=f"IVF{nlist},PQ{M}+{M2}", dim=d, metric="l2",
                       train_num=1000, nprobe=3, index_format="faiss")
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
            assert ix.faiss_index.kind == 6 and ix.faiss_index.nprobe == 3 and ix.faiss_index.metric == L2
            st = ix.faiss_index.get_state()
            before.append(st)
            o = OracleIVFPQR(d, nlist, M, M2)
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
        for s, st in zip(servers, before):
            after = s.indexes[index_id].faiss_index.get_state()
            for key in STATE_KEYS:
                assert np.asarray(after[key]).tobytes() == np.asarray(st[key]).tobytes(), key
        D1, M1 = c2.search(xq, k, index_id)
        assert np.array_equal(np.asarray(D1, dtype=np.float32), refD) and M1 == meta
        c2.close()
    finally:
        for s in servers:
            s.stop()
