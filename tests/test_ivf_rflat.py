"""Flat refinement ("IVF{n},<codec>,RFlat"): the k * k_factor best candidates of a codec shard re-ranked
on their stored fp32 vectors (dfx_rflat_dev.cuh).

CPU: the factory parser, the oracle against a float64 restatement, persistence (npz and the faiss
format "IxRF") and sharded search through the servers with oracle engines; this file's `gpu` tests
also run against the emulated library.
GPU: the CUDA kernels against the oracle, bit for bit, for the four base kinds and the three k'
regimes (queues, candidate rows, k' > 4096); the equality with an IVF-Flat shard when every probed
vector is re-ranked; adds after a search; state export -> import; graph-captured shard groups; the
servers / client end to end over sockets and over the search plane."""
import os
import platform
import shutil
import subprocess
import sys
import tempfile
import threading
import time

import numpy as np
import pytest

from tests.conftest import clustered

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
IP, L2 = 0, 1
FMAX = np.finfo(np.float32).max
EMU = bool(os.environ.get("DFX_EMU_LIB"))
CODECS = {"ivf_pq": "PQ{M}", "ivf_pq_fs": "PQ{M}x4fs", "ivf_sq8": "SQ8", "ivf_sq": "SQfp16"}
PAYLOAD = {"ivf_pq": "codes", "ivf_pq_fs": "codes", "ivf_sq8": "codes8", "ivf_sq": "codes16"}


def _sz(full, emu):
    return emu if EMU else full


@pytest.fixture
def rflat_oracle(oracle_lib):
    """(kind, d, nlist, M, n, seed) -> a trained, filled oracle shard with a flat refinement, and its rows"""
    from tests.oracle_rflat import make_rflat

    def make(kind, d=64, nlist=8, M=8, n=1500, seed=0, niter=4):
        rs = np.random.RandomState(seed)
        o = make_rflat(kind, d, nlist, M)
        o.train_niter = niter
        xb = clustered(rs, n, d, ncl=max(4, nlist // 2))
        o.train(xb)
        o.add(xb[: n // 3])
        o.add(xb[n // 3:])
        return o, xb

    return make


# ------------------------------------------------------------------ parser, CPU
@pytest.mark.parametrize("s,kind,M", [("IVF4096,PQ16,RFlat", "ivf_pq", 16), ("IVF4096,PQ128x8,RFlat", "ivf_pq", 128),
                                      ("IVF4096,PQ32x4fs,RFlat", "ivf_pq_fs", 32), ("IVF4096,SQ8,RFlat", "ivf_sq8", 0),
                                      ("IVF4096,SQfp16,RFlat", "ivf_sq", 0)])
def test_parser_accepts_rflat(s, kind, M):
    from distributed_faiss_b200.factory import ACCEPTED_FORMS, FactorySpec, parse_factory

    spec = parse_factory(128, s, L2)
    assert spec == FactorySpec(kind, L2, 4096, M, 0, True) and spec.refine_flat is True
    plain = parse_factory(128, s[:-len(",RFlat")], L2)
    assert plain == FactorySpec(kind, L2, 4096, M) and plain.refine_flat is False   # the default stays off
    for form in ("IVF{n},PQ{M},RFlat", "IVF{n},PQ{M}x8,RFlat", "IVF{n},PQ{M}x4fs,RFlat", "IVF{n},SQ8,RFlat",
                 "IVF{n},SQfp16,RFlat"):
        assert form in ACCEPTED_FORMS


@pytest.mark.parametrize("s", [
    "IVF64,Flat,RFlat", "Flat,RFlat", "IVF64,PQ16,Refine(Flat)", "IVF64,SQ8,Refine(SQ8)", "IVF64,PQ16,Refine(PQ16)",
    "IVF64,PQ16+16,RFlat", "IVF64,PQ16x4fsr", "IVF64,PQ16x4fsr,RFlat", "IVF64,PQ16x4fs_64", "IVF64,PQ16x4fs_64,RFlat",
    "IVF64,PQ16x4", "IVF64,PQ16x4,RFlat", "IVF64,PQ16,RFlat,", "IVF64,PQ16,rflat", "IVF64,PQ16,RFlat,RFlat",
    "IVF64,RFlat", "RFlat",
])
def test_parser_refuses_the_other_refinements(s):
    from distributed_faiss_b200.factory import ACCEPTED_FORMS, parse_factory

    with pytest.raises(RuntimeError, match="not supported") as e:
        parse_factory(64, s, L2)
    assert repr(s) in str(e.value) and all(f in str(e.value) for f in ACCEPTED_FORMS)


def test_parser_keeps_the_codec_limits_and_the_inner_product_message():
    from distributed_faiss_b200.factory import parse_factory
    from distributed_faiss_b200.index import factory_spec
    from distributed_faiss_b200.index_cfg import IndexCfg

    for s in ("IVF64,PQ16,RFlat", "IVF64,PQ16x4fs,RFlat", "IVF64,SQ8,RFlat", "IVF64,SQfp16,RFlat"):
        with pytest.raises(RuntimeError, match="inner-product distance tables"):
            parse_factory(64, s, IP)
    with pytest.raises(RuntimeError, match="multiple of 4"):
        parse_factory(64, "IVF64,PQ6,RFlat", L2)
    with pytest.raises(RuntimeError, match="multiple of 8"):
        parse_factory(96, "IVF64,PQ12x4fs,RFlat", L2)
    with pytest.raises(RuntimeError, match="inner-product distance tables"):
        factory_spec(IndexCfg(faiss_factory="IVF{centroids},PQ16x4fs,RFlat", dim=64, centroids=8, metric="dot"))
    # ivf_gpu: the raw string and faiss's default metric, L2, whatever cfg.metric says
    cfg = IndexCfg(index_builder_type="ivf_gpu", faiss_factory="IVF16,PQ8x4fs,RFlat", dim=64, metric="dot", nprobe=3)
    spec = factory_spec(cfg)
    assert (spec.kind, spec.metric, spec.pq_m, spec.refine_flat) == ("ivf_pq_fs", L2, 8, True)


# ------------------------------------------------------------------ oracle, CPU
@pytest.mark.parametrize("kind", list(CODECS))
def test_oracle_matches_warp_dot_and_a_float64_restatement(kind, rflat_oracle):
    """each distance is oracle.warp_dot's L2 of (q, stored row) and within fp32 rounding of float64
    |q - x|^2; the ids are those of float64 wherever its distances are further apart than that"""
    from oracle import oracle as O
    from tests.oracle_rflat import BASES, exact_f64

    o, xb = rflat_oracle(kind, seed=1)
    o.nprobe, o.k_factor, k = 3, 4.0, 10
    xq = np.concatenate([clustered(np.random.RandomState(2), 12, 64, ncl=8), xb[:4] + np.float32(0.01)])
    D, I = o.search(xq, k)
    _, I1 = BASES[kind].search(o, xq, 4 * k)   # the first stage's candidates
    assert np.array_equal(o.refine_vecs, xb)
    for q in range(len(xq)):
        cand = I1[q][I1[q] >= 0]
        assert set(I[q][I[q] >= 0].tolist()) <= set(cand.tolist())
        exact = exact_f64(xq[q:q + 1], xb, cand)[0]
        tol = 1e-5 * (exact.max() + (xq[q].astype(np.float64) ** 2).sum() + 1)
        got = dict(zip(I[q].tolist(), D[q].tolist()))
        for i, e in zip(cand.tolist(), exact.tolist()):
            if i in got:
                assert got[i] == O.warp_dot(xq[q], xb[i], 1) and abs(got[i] - e) <= tol, (q, i)
        kth = np.sort(exact)[min(k, len(exact)) - 1]
        assert set(cand[exact < kth - 2 * tol].tolist()) <= set(I[q].tolist()), q
        assert all(e <= kth + 2 * tol for i, e in zip(cand.tolist(), exact.tolist()) if i in got), q
    ids = np.array([0, 7, -1, len(xb) - 1])
    R = o.reconstruct_rows(ids)
    assert np.isnan(R[2]).all() and np.array_equal(R[[0, 1, 3]], xb[[0, 7, len(xb) - 1]])


def _recall(I, gt):
    return np.mean([len(set(a.tolist()) & set(b.tolist())) / gt.shape[1] for a, b in zip(I, gt)])


def test_refinement_raises_recall_on_clustered_data(rflat_oracle):
    """the point of the feature: FastScan's 4-bit codes with an exact re-rank of 4k candidates find
    more of the true neighbours than the codes alone, and never more than IVF-Flat at the same nprobe"""
    from oracle import oracle as O
    from tests.oracle_rflat import BASES

    o, xb = rflat_oracle("ivf_pq_fs", d=64, nlist=16, M=8, n=4000, seed=3)
    o.nprobe, k = 4, 10
    xq = clustered(np.random.RandomState(4), 100, 64, ncl=8)
    _, gt = O.flat_search(L2, xb, xq, k)
    _, I_fs = BASES["ivf_pq_fs"].search(o, xq, k)
    o.k_factor = 4.0
    _, I_rf = o.search(xq, k)
    flat = O.OracleIVFFlat(64, 16, L2)
    flat.set_state(dict(centroids=o.centroids, list_off=o.list_off, ids=o.ids, vecs=xb[o.ids]))
    flat.nprobe = 4
    _, I_flat = flat.search(xq, k)
    r_fs, r_rf, r_flat = _recall(I_fs, gt), _recall(I_rf, gt), _recall(I_flat, gt)
    assert r_fs + 0.05 < r_rf <= r_flat, (r_fs, r_rf, r_flat)


# ------------------------------------------------------------------ persistence / servers, CPU
def _cfg(kind, d, M=8, **kw):
    from distributed_faiss_b200.index_cfg import IndexCfg

    return IndexCfg(faiss_factory="IVF{centroids}," + CODECS[kind].format(M=M) + ",RFlat", dim=d, metric="l2", **kw)


def _wait_trained_index(ix):
    from distributed_faiss_b200.index_state import IndexState

    t0 = time.time()
    while ix.get_state() != IndexState.TRAINED:
        assert time.time() - t0 < 60, "index never reached TRAINED"
        time.sleep(0.01)


def _same_state(a, b, kind):
    for key in ("centroids", "list_off", "ids", PAYLOAD[kind], "refine_vecs"):
        assert np.asarray(a[key]).tobytes() == np.asarray(b[key]).tobytes(), key
    assert a["refine_flat"] == b["refine_flat"] == 1 and a["k_factor"] == b["k_factor"]


@pytest.mark.parametrize("kind", ["ivf_pq", "ivf_sq8", "ivf_sq"])
def test_ixrf_round_trip(kind, rflat_oracle, tmp_path):
    from distributed_faiss_b200 import faiss_io

    o, xb = rflat_oracle(kind, d=32, nlist=6, n=500, seed=5)
    o.k_factor = 2.5
    st = o.get_state()
    path = str(tmp_path / "rf.faiss")
    faiss_io.write_index(st, path, nprobe=3)
    raw = open(path, "rb").read()
    assert raw[:4] == b"IxRF" and raw[-4:] == np.float32(2.5).tobytes()
    back, nprobe = faiss_io.read_index(path)
    assert nprobe == 3 and back["kind"] == kind
    _same_state(st, back, kind)
    # the same shard without the refinement is written as the base index alone, exactly as before
    plain = {k: v for k, v in st.items() if k not in ("refine_flat", "refine_vecs", "k_factor")}
    faiss_io.write_index(plain, str(tmp_path / "plain.faiss"), nprobe=3)
    base = open(str(tmp_path / "plain.faiss"), "rb").read()
    assert base[:2] == b"Iw" and base in raw and "refine_flat" not in faiss_io.read_index(str(tmp_path / "plain.faiss"))[0]
    # a refine index that does not hold ntotal rows is refused, and so is a truncated file
    with pytest.raises(faiss_io.FaissFormatError, match="ntotal vectors"):
        faiss_io.write_index(dict(st, refine_vecs=st["refine_vecs"][:-1]), str(tmp_path / "bad.faiss"))
    with open(str(tmp_path / "cut.faiss"), "wb") as f:
        f.write(raw[:-8])
    with pytest.raises(faiss_io.FaissFormatError):
        faiss_io.read_index(str(tmp_path / "cut.faiss"))


def test_ixrf_is_refused_around_fastscan_and_unserved_bases(rflat_oracle, tmp_path):
    from distributed_faiss_b200 import faiss_io
    from oracle import oracle as O

    o, _ = rflat_oracle("ivf_pq_fs", d=32, nlist=6, n=300, seed=6)
    with pytest.raises(faiss_io.FaissFormatError, match="IndexIVFPQFastScan"):
        faiss_io.write_index(o.get_state(), str(tmp_path / "fs.faiss"))
    flat = O.OracleFlat(8, L2)
    flat.add(np.zeros((3, 8), np.float32))
    with pytest.raises(faiss_io.FaissFormatError, match="kind 'flat' is not served"):
        faiss_io.write_index(dict(flat.get_state(), refine_flat=1, refine_vecs=np.zeros((3, 8), np.float32), ids=np.arange(3)),
                             str(tmp_path / "flat.faiss"))
    # IxRF around a flat index, as faiss writes "Flat,RFlat": read as far as the base, then refused
    with open(str(tmp_path / "f.faiss"), "wb") as f:
        f.write(b"IxRF")
        faiss_io._wheader(f, 8, 3, L2)
        faiss_io._write_flat(f, np.zeros((3, 8), np.float32), L2)
        faiss_io._write_flat(f, np.zeros((3, 8), np.float32), L2)
        faiss_io._w(f, "f", 1.0)
    with pytest.raises(faiss_io.FaissFormatError, match="kind 'flat'"):
        faiss_io.read_index(str(tmp_path / "f.faiss"))


def test_rflat_shard_through_index_with_k_factor_embeddings_and_saved_files(oracle_lib, tmp_path):
    from distributed_faiss_b200.index import Index
    from distributed_faiss_b200.index_cfg import IndexCfg
    from tests.oracle_rflat import BASES, oracle_engine_factory

    rs = np.random.RandomState(7)
    d, nlist = 32, 6
    x = clustered(rs, 600, d, ncl=6)
    q = x[::60] + np.float32(0.01)
    for kind, fmt in (("ivf_pq_fs", "dfx"), ("ivf_pq", "faiss"), ("ivf_sq8", "dfx"), ("ivf_sq", "faiss")):
        root = tmp_path / f"{kind}_{fmt}"
        os.makedirs(root)
        cfg = _cfg(kind, d, centroids=nlist, train_num=400, index_storage_dir=str(root), index_format=fmt, k_factor=3)
        ix = Index(cfg, engine_factory=oracle_engine_factory)
        for b in range(3):   # several batches; the last two are added after training
            ix.add_batch(x[200 * b:200 * (b + 1)], [("m", i) for i in range(200 * b, 200 * (b + 1))],
                         train_async_if_triggered=False)
            if b:
                _wait_trained_index(ix)
        t0 = time.time()
        while ix.faiss_index.ntotal != 600:
            assert time.time() - t0 < 60
            time.sleep(0.01)
        _wait_trained_index(ix)
        o = ix.faiss_index
        assert isinstance(o, BASES[kind]) and o.refine_flat and o.k_factor == 3.0 and o.nprobe == 1
        ix.set_nprobe(3)
        D1, m1, E1 = ix.search(q, 7, return_embeddings=True)
        # the embeddings are the raw rows (metadata ("m", i) names row i), not the codec's decode
        for qi in range(len(q)):
            for j, m in enumerate(m1[qi]):
                if m is not None:
                    assert np.array_equal(E1[qi][j], x[m[1]])
        assert ix.save()
        assert os.path.isfile(root / ("index.faiss" if fmt == "faiss" else "index.dfx.npz"))
        cfg2 = IndexCfg.from_json(str(root / "cfg.json"))
        assert cfg2.extra["k_factor"] == 3
        ix2 = Index.from_storage_dir(str(root), cfg2, engine_factory=oracle_engine_factory)
        ix2.set_nprobe(3)
        _same_state(o.get_state(), ix2.faiss_index.get_state(), kind)
        D2, m2, _ = ix2.search(q, 7)
        assert D1.tobytes() == D2.tobytes() and m1 == m2
        # a cfg that carries another k_factor wins over the stored one; one that carries none keeps it
        cfg3 = IndexCfg.from_json(str(root / "cfg.json"))
        cfg3.extra["k_factor"] = 5
        assert Index.from_storage_dir(str(root), cfg3, engine_factory=oracle_engine_factory).faiss_index.k_factor == 5.0
        del cfg3.extra["k_factor"]
        assert Index.from_storage_dir(str(root), cfg3, engine_factory=oracle_engine_factory).faiss_index.k_factor == 3.0

        def gpu_cfg(s):
            return IndexCfg(index_builder_type="ivf_gpu", faiss_factory=s, dim=d, metric="l2")

        codec = CODECS[kind].format(M=8)
        with pytest.raises(RuntimeError, match=rf"{kind!r} with a flat refinement \(RFlat\) but the cfg builds {kind!r}; "):
            Index.from_storage_dir(str(root), gpu_cfg(f"IVF{nlist},{codec}"), engine_factory=oracle_engine_factory)
        other = "SQ8" if kind != "ivf_sq8" else "SQfp16"
        with pytest.raises(RuntimeError, match="refusing to load it"):
            Index.from_storage_dir(str(root), gpu_cfg(f"IVF{nlist},{other},RFlat"), engine_factory=oracle_engine_factory)
        ix4 = Index.from_storage_dir(str(root), gpu_cfg(f"IVF{nlist},{codec},RFlat"), engine_factory=oracle_engine_factory)
        assert ix4.faiss_index.get_state()["refine_vecs"].shape == (600, d)
    # and a shard stored without the refinement is refused under a cfg that builds one
    root = tmp_path / "plain"
    os.makedirs(root)
    cfg = IndexCfg(faiss_factory="IVF{centroids},SQ8", dim=d, metric="l2", centroids=nlist, train_num=400,
                   index_storage_dir=str(root))
    ix = Index(cfg, engine_factory=oracle_engine_factory)
    ix.add_batch(x, None, train_async_if_triggered=False)
    _wait_trained_index(ix)
    t0 = time.time()
    while ix.faiss_index.ntotal != 600:
        assert time.time() - t0 < 60
        time.sleep(0.01)
    _wait_trained_index(ix)
    assert ix.save()
    with pytest.raises(RuntimeError, match=r"'ivf_sq8' but the cfg builds 'ivf_sq8' with a flat refinement \(RFlat\)"):
        Index.from_storage_dir(str(root), gpu_cfg(f"IVF{nlist},SQ8,RFlat"), engine_factory=oracle_engine_factory)


def test_rflat_sharded_search_is_the_merge_of_the_shards(oracle_lib):
    from distributed_faiss_b200.client import ResultHeap
    from distributed_faiss_b200.index_state import IndexState
    from distributed_faiss_b200.server import IndexServer
    from oracle import oracle as O
    from tests.oracle_engine import oracle_merge
    from tests.oracle_rflat import oracle_engine_factory
    from tests.test_host_logic import free_ports, make_client, wait_listening, wait_trained

    ResultHeap.merge_backend = staticmethod(oracle_merge)
    tmp = tempfile.TemporaryDirectory()
    ports = free_ports(2)
    servers = [IndexServer(r, tmp.name, engine_factory=oracle_engine_factory) for r in range(2)]
    for s, p in zip(servers, ports):
        threading.Thread(target=s.start_blocking, args=(p,), daemon=True).start()
    wait_listening(ports)
    try:
        rs = np.random.RandomState(8)
        d, nlist, k = 64, 8, 12
        client = make_client(ports)
        client.create_index("rf", _cfg("ivf_pq_fs", d, M=16, centroids=nlist, train_num=600, k_factor=4))
        xs = [clustered(rs, 400, d, ncl=8) for _ in range(6)]
        for b, x in enumerate(xs):
            client.add_index_data("rf", x, list(range(400 * b, 400 * (b + 1))), False)
        client.sync_train("rf")
        wait_trained(client, "rf")
        t0 = time.time()
        while client.get_ntotal("rf") != 2400 or client.get_state("rf") != IndexState.TRAINED:
            assert time.time() - t0 < 60, "adds never finished"
            time.sleep(0.02)
        client.set_nprobe("rf", 3)
        allx = np.concatenate(xs)
        xq = allx[::101][:12] + np.float32(0.01)
        D, meta, embs = client.search(xq, k, "rf", return_embeddings=True)
        Ds, Ps, metas = [], [], []
        for s in servers:
            ix = s.indexes["rf"]
            assert ix.faiss_index.kind == "ivf_pq_fs" and ix.faiss_index.refine_flat and ix.faiss_index.k_factor == 4.0
            Do, Io = ix.faiss_index.search(xq, k)
            Ds.append(Do); Ps.append(Io); metas.append(ix.id_to_metadata)
        Dall = np.stack(Ds)
        pos = np.arange(Dall.size, dtype=np.int64).reshape(Dall.shape)
        refD, refP = O.merge(Dall, pos)
        assert np.array_equal(np.asarray(D, dtype=np.float32), refD)
        S_, nq_, k_ = Dall.shape
        want = [[metas[p // (nq_ * k_)][int(Ps[p // (nq_ * k_)][q, p % k_])] for p in refP[q]] for q in range(nq_)]
        assert [list(r) for r in meta] == want
        for q in range(nq_):   # metadata i names row i of everything that was added
            for j, m in enumerate(meta[q]):
                assert np.array_equal(np.asarray(embs[q][j], dtype=np.float32), allx[m])
        client.close()
    finally:
        for s in servers:
            s.stop()


# ------------------------------------------------------------------ the gpu tests on the emulator
EMU_SUBSET = [
    "tests/test_ivf_rflat.py::test_rflat_matches_oracle",
    "tests/test_ivf_rflat.py::test_rflat_equals_ivf_flat_when_every_probed_vector_is_reranked",
    "tests/test_ivf_rflat.py::test_rflat_adds_after_a_search_and_state_round_trip",
    "tests/test_ivf_rflat.py::test_rflat_limits",
]


def test_rflat_gpu_tests_on_the_emulated_library():
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
    assert " passed" in run.stdout and "failed" not in run.stdout, tail


# ------------------------------------------------------------------ GPU parity
def _assert_same(Dg, Ig, Do, Io, what):
    if not (np.array_equal(Ig, Io) and np.array_equal(Dg, Do)):
        bad = np.argwhere((Ig != Io) | (Dg != Do))
        q, j = bad[0]
        raise AssertionError(f"{what}: {len(bad)} mismatching slots of {Ig.size}; first at q={q} j={j}: "
                             f"gpu=({Dg[q, j]!r},{Ig[q, j]}) oracle=({Do[q, j]!r},{Io[q, j]})")


def _gpu(kind, d, nlist, M=0, **kw):
    from distributed_faiss_b200 import engine as E

    k = {name: n for n, name in E.KIND_NAMES.items()}[kind]
    return E.GpuIndex(k, d, L2, nlist=nlist, pq_m=M, pq_nbits=4 if kind == "ivf_pq_fs" else 8, refine_flat=True, **kw)


def _build_both(kind, d, nlist, M, n, rs, via):
    """a GPU shard and the oracle holding the same state: built on the GPU and exported, or trained by
    the oracle and imported"""
    from tests.oracle_rflat import make_rflat

    xb = clustered(rs, n, d, ncl=max(8, nlist // 2))
    g, o = _gpu(kind, d, nlist, M), make_rflat(kind, d, nlist, M)
    assert g.get_param("k_factor") == 1.0   # faiss IndexRefine default
    if via == "gpu":
        g.set_param("kmeans_niter", 2)
        g.train(xb[: n // 2])
        g.add(xb[: n // 3]); g.add(xb[n // 3:])
        st = g.get_state()
        assert st["kind"] == kind and st["refine_flat"] == 1 and st["k_factor"] == 1.0
        assert np.array_equal(st["refine_vecs"], xb)    # the raw rows, in id (arrival) order
        o.set_state(st)
    else:
        o.train_niter = 2
        o.train(xb[: n // 2])
        o.add(xb)
        g.set_state(o.get_state())
        assert np.array_equal(g.get_array("refine_vecs").reshape(-1, d), xb)
    assert g.ntotal == n == o.ntotal
    return g, o, xb


CASES = [("ivf_pq", 128, 16), ("ivf_pq", 128, 32), ("ivf_pq", 192, 96), ("ivf_pq_fs", 128, 32), ("ivf_pq_fs", 64, 16),
         ("ivf_sq8", 128, 0), ("ivf_sq", 96, 0), ("ivf_sq", 320, 0)]


@pytest.mark.gpu
@pytest.mark.parametrize("kind,d,M", CASES)
@pytest.mark.parametrize("via", ["gpu", "oracle"])
def test_rflat_matches_oracle(kind, d, M, via):
    """distances, ids and ndis bit for bit for k in {1, 10, 100} and k_factor in {1, 4}, then the three
    k' regimes: k' <= 1024 (queues), 1024 < k' <= 4096 (candidate rows) and 4096 < k' <= 16384.
    M = 32 is the interleaved scan, M = 96 the wide one; d = 320 rows are longer than 1 KB"""
    if EMU and (via == "oracle") != (kind == "ivf_sq8" or (kind, M) == ("ivf_pq", 16)):
        pytest.skip("one build path per case on the emulator")
    rs = np.random.RandomState(20)
    nlist = 16
    g, o, xb = _build_both(kind, d, nlist, M, _sz(6000, 1000), rs, via)
    if (kind, M) == ("ivf_pq", 32):
        assert g.get_param("interleaved") == 1
    xq = np.concatenate([clustered(rs, _sz(10, 3), d, ncl=8), xb[:3] + 0.01 * rs.randn(3, d).astype(np.float32)])
    for nprobe in (nlist, 1, 5):   # all lists; one (fewer than k hits); several probe groups per query
        g.nprobe = o.nprobe = nprobe
        for k_factor, ks in ((1, (1, 10, 100)), (4, (1, 10, 100) if EMU else (1, 10, 100, 256, 257, 1024, 1025, 4096))):
            g.set_param("k_factor", k_factor)
            o.k_factor = k_factor
            for k in ks:
                Dg, Ig = g.search(xq, k)
                Do, Io = o.search(xq, k)
                _assert_same(Dg, Ig, Do, Io, f"{kind} M={M} d={d} via={via} nprobe={nprobe} k_factor={k_factor} k={k}")
                assert g.last_stats()["ndis"] == o.last_ndis
        if nprobe == 1:   # fewer than k hits: padded with (FLT_MAX, -1)
            g.set_param("k_factor", 1)
            o.k_factor = 1.0
            Dg, Ig = g.search(xq, _sz(4096, 600))
            _assert_same(Dg, Ig, *o.search(xq, _sz(4096, 600)), f"{kind} fewer than k hits")
            assert (Ig == -1).any() and (Dg[Ig == -1] == FMAX).all()
    ids = np.array([0, 5, len(xb) - 1, -1, 17], dtype=np.int64)
    R = g.reconstruct_rows(ids)
    assert np.isnan(R[3]).all() and np.array_equal(R[[0, 1, 2, 4]], xb[[0, 5, len(xb) - 1, 17]])
    Dg, Ig, Rg = g.search_and_reconstruct(xb[:4], 5)
    assert np.array_equal(Rg[Ig >= 0], xb[Ig[Ig >= 0]])


@pytest.mark.gpu
@pytest.mark.parametrize("kind,d,M", [("ivf_pq", 64, 8), ("ivf_pq_fs", 64, 8), ("ivf_sq8", 64, 0), ("ivf_sq", 64, 0)])
def test_rflat_equals_ivf_flat_when_every_probed_vector_is_reranked(kind, d, M):
    """metamorphic: with k' at least the number of probed vectors the first stage drops nothing, so the
    answer is, bit for bit, that of an IVF-Flat L2 shard holding the same centroids, lists and rows"""
    from distributed_faiss_b200 import engine as E

    rs = np.random.RandomState(21)
    nlist, n = 8, _sz(3000, 900)
    g, o, xb = _build_both(kind, d, nlist, M, n, rs, "gpu")
    st = g.get_state()
    flat = E.GpuIndex(E.KIND_IVF_FLAT, d, L2, nlist=nlist)
    flat.set_state({"centroids": st["centroids"], "list_off": st["list_off"], "ids": st["ids"], "vecs": xb[st["ids"]]})
    xq = np.concatenate([clustered(rs, 6, d, ncl=8), xb[:2] + np.float32(0.01)])
    for nprobe, k, k_factor in ((3, 100, 30), (nlist, 100, 30), (1, 10, 300), (2, 1000, 3)):
        assert int(np.float32(k) * np.float32(k_factor)) >= n
        g.nprobe = flat.nprobe = nprobe
        g.set_param("k_factor", k_factor)
        Dg, Ig = g.search(xq, k)
        Df, If = flat.search(xq, k)
        _assert_same(Dg, Ig, Df, If, f"{kind} nprobe={nprobe} k={k}")
        assert g.last_stats()["ndis"] == flat.last_stats()["ndis"]


@pytest.mark.gpu
def test_rflat_adds_after_a_search_and_state_round_trip():
    """adds append to the refinement store across a search (and a regrowth of the store); an exported
    state imported into a fresh shard answers with the same bits, k_factor included"""
    rs = np.random.RandomState(22)
    d, nlist, M = 64, 8, 16
    g, o, xb = _build_both("ivf_pq_fs", d, nlist, M, _sz(2000, 600), rs, "gpu")
    g.nprobe = o.nprobe = 3
    g.set_param("k_factor", 4); o.k_factor = 4.0
    xq = xb[:5] + np.float32(0.01)
    _assert_same(*g.search(xq, 10), *o.search(xq, 10), "before the adds")
    for _ in range(3):
        more = clustered(rs, _sz(1500, 500), d, ncl=8)
        g.add(more); o.add(more)
        xb = np.concatenate([xb, more])
        _assert_same(*g.search(xq, 10), *o.search(xq, 10), "after an add")
    st = g.get_state()
    assert np.array_equal(st["refine_vecs"], xb) and st["k_factor"] == 4.0
    g2 = _gpu("ivf_pq_fs", d, nlist, M)
    g2.set_state(st)
    g2.nprobe = 3
    assert g2.get_param("k_factor") == 4.0
    for k in (1, 10, 300):
        _assert_same(*g2.search(xq, k), *g.search(xq, k), f"imported shard k={k}")
    st2 = g2.get_state()
    for key in ("centroids", "codebooks", "list_off", "ids", "codes", "refine_vecs"):
        assert np.asarray(st[key]).tobytes() == np.asarray(st2[key]).tobytes(), key
    assert np.array_equal(g2.reconstruct_rows(np.arange(0, len(xb), 97)), xb[::97])


@pytest.mark.gpu
def test_rflat_limits(rflat_oracle):
    from distributed_faiss_b200 import engine as E

    for kind, M in (("ivf_pq", 128), ("ivf_pq_fs", 8), ("ivf_sq8", 0), ("ivf_sq", 0)):
        _gpu(kind, 256, 4, M)
    with pytest.raises(RuntimeError, match="refine_flat must be 0 for FLAT and IVF_FLAT"):
        E.GpuIndex(E.KIND_FLAT, 64, L2, refine_flat=True)
    with pytest.raises(RuntimeError, match="refine_flat must be 0 for FLAT and IVF_FLAT"):
        E.GpuIndex(E.KIND_IVF_FLAT, 64, L2, nlist=4, refine_flat=True)
    with pytest.raises(RuntimeError, match="refine_flat must be 0 for IVF_PQR"):
        E.GpuIndex(E.KIND_IVF_PQR, 64, L2, nlist=4, pq_m=8, refine_m=8, refine_flat=True)
    with pytest.raises(RuntimeError, match="refine_flat must be 0 for IVF-PQ with 4-bit codes"):
        E.GpuIndex(E.KIND_IVF_PQ, 64, L2, nlist=4, pq_m=8, pq_nbits=4, refine_flat=True)
    with pytest.raises(RuntimeError, match="flat refinement: only the L2 metric"):
        E.GpuIndex(E.KIND_IVF_SQ8, 64, IP, nlist=4, refine_flat=True)
    o, xb = rflat_oracle("ivf_sq8", d=64, nlist=4, n=300, seed=23)
    st = o.get_state()
    g = _gpu("ivf_sq8", 64, 4)
    for bad in (0.5, 0, -1, 16385):
        with pytest.raises(RuntimeError, match=r"k_factor must be in \[1, 16384\]"):
            g.set_param("k_factor", bad)
    plain = E.GpuIndex(E.KIND_IVF_SQ8, 64, L2, nlist=4)
    with pytest.raises(RuntimeError, match="k_factor is a parameter of IVF-PQR"):
        plain.set_param("k_factor", 2)
    with pytest.raises(RuntimeError, match="unknown parameter k_factor"):
        plain.get_param("k_factor")
    with pytest.raises(RuntimeError, match="no array named 'refine_vecs'"):
        plain.get_array("refine_vecs")
    g.set_state(st)
    # a k' beyond 16384 raises before anything is launched, naming k and k_factor
    g.set_param("k_factor", 4.5)
    n0 = E.launch_count()
    with pytest.raises(RuntimeError, match=r"k=4096 with k_factor=4\.5.*18432 candidates to re-rank, more than 16384"):
        g.search(st["centroids"][:2], 4096)
    with pytest.raises(RuntimeError, match="IVF search supports k <= 4096"):
        g.search(st["centroids"][:2], 4097)
    assert E.launch_count() == n0
    g.set_param("k_factor", 4)
    g.nprobe = 4
    D, I = g.search(st["centroids"][:2], 4096)   # k' = 16384, every list probed
    assert (I[:, 300:] == -1).all() and (I[:, :300] >= 0).all()
    # the rows are addressed by id: the ids of an import must be a permutation, the store must be whole
    bad = st["ids"].copy()
    bad[[3, 4]] = bad[3]
    g2 = _gpu("ivf_sq8", 64, 4)
    with pytest.raises(RuntimeError, match="permutation"):
        g2.set_state(dict(st, ids=bad))
    with pytest.raises(RuntimeError, match="refine_vecs: wrong size"):
        g2.set_state(dict(st, refine_vecs=st["refine_vecs"][:-1]))
    with pytest.raises(RuntimeError, match=r"sq_trained: wrong size \(2 \* d floats"):
        g2.set_array("sq_trained", st["sq_trained"][:1])
    from tests.test_gpu_parity import _import_without

    for skip, msg in (("sq_trained", "sq_trained is required"), ("refine_vecs", "refine_vecs of every vector are required")):
        with pytest.raises(RuntimeError, match="import: " + msg):
            _import_without(_gpu("ivf_sq8", 64, 4), st, skip)


@pytest.mark.gpu
def test_rflat_many_queries_and_the_refine_stage_timer():
    """a batch of more queries than one re-ranking chunk (qc * k' <= 2^22), and refine_ms / refine_launches"""
    if EMU:
        pytest.skip("too large for the emulator")
    rs = np.random.RandomState(24)
    d, nlist, M = 128, 16, 32
    g, o, xb = _build_both("ivf_pq_fs", d, nlist, M, 6000, rs, "oracle")
    g.nprobe = o.nprobe = nlist
    g.set_param("k_factor", 4); o.k_factor = 4.0
    QC = (1 << 22) // 4100                # the re-ranking chunk at k' = 4 * 1025
    xq = clustered(rs, QC + 300, d, ncl=8)
    g.profile(True)
    Dg, Ig = g.search(xq, 1025)
    assert g.get_param("refine_launches") == 2 and g.get_param("refine_ms") > 0
    scan_ms, scans = g.profile_read(reset=True)
    assert scans == 2 and scan_ms > 0 and g.get_param("refine_launches") == 0
    g.profile(False)
    rows = np.array([0, 1, QC - 1, QC, QC + 1, len(xq) - 1])
    Do, Io = o.search(xq[rows], 1025)
    _assert_same(Dg[rows], Ig[rows], Do, Io, "chunk edges")
    Dg, Ig = g.search(xq, 10)
    Do, Io = o.search(xq[rows], 10)
    _assert_same(Dg[rows], Ig[rows], Do, Io, "k=10 batch")


@pytest.mark.gpu
def test_rflat_device_paths_match_the_host_path(monkeypatch):
    """search_dev equals search; a ShardGroup of refined shards replays its search from a captured CUDA
    graph with the eager answers"""
    if EMU:
        pytest.skip("CUDA tensors")
    import torch

    from distributed_faiss_b200 import spmd

    rs = np.random.RandomState(25)
    shards, tables, base = [], [], 0
    for kind, M in (("ivf_pq_fs", 32), ("ivf_pq", 32), ("ivf_sq8", 0)):
        g, o, xb = _build_both(kind, 128, 32, M, 8000, rs, "gpu")
        g.nprobe = 6
        g.set_param("k_factor", 4)
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


@pytest.mark.gpu
@pytest.mark.parametrize("builder", ["factory", "ivf_gpu"])
def test_rflat_through_the_client_over_sockets_and_the_plane(builder):
    """two IndexServers on the GPU engine, "IVF8,PQ32x4fs,RFlat" with k_factor = 4 from the cfg: the
    client's merged answer with embeddings is the merge of the oracle's answers on each shard, over the
    socket fan-out and over the search plane, and a saved index loads back to the same state and bits"""
    if EMU:
        pytest.skip("CUDA tensors")
    from distributed_faiss_b200.index_cfg import IndexCfg
    from oracle import oracle as O
    from tests.oracle_rflat import make_rflat
    from tests.test_gpu_api import _plane_cluster, make_client

    store, servers, plane, client = _plane_cluster(2)
    try:
        rs = np.random.RandomState(26)
        d, nlist, M, k, index_id = 128, 8, 32, 20, "rf"
        if builder == "factory":
            cfg = IndexCfg(faiss_factory="IVF{centroids},PQ32x4fs,RFlat", dim=d, metric="l2", centroids=nlist,
                           train_num=1000, k_factor=4)
        else:
            cfg = IndexCfg(index_builder_type="ivf_gpu", faiss_factory=f"IVF{nlist},PQ32x4fs,RFlat", dim=d, metric="l2",
                           train_num=1000, nprobe=3, k_factor=4)
        client.create_index(index_id, cfg)
        xs = [clustered(rs, 1000, d, ncl=8) for _ in range(4)]
        for b, x in enumerate(xs):
            client.add_index_data(index_id, x, list(range(1000 * b, 1000 * (b + 1))), False)
        client.sync_train(index_id)
        t0 = time.time()
        from distributed_faiss_b200.index_state import IndexState
        while client.get_ntotal(index_id) != 4000 or client.get_state(index_id) != IndexState.TRAINED:
            assert time.time() - t0 < 300, "adds never finished"
            time.sleep(0.05)
        client.set_nprobe(index_id, 3)
        allx = np.concatenate(xs)
        xq = allx[::211][:16] + np.float32(0.01)
        Ds, Ps, metas, before = [], [], [], []
        for s in servers:
            ix = s.indexes[index_id]
            assert ix.faiss_index.kind == 5 and ix.faiss_index.refine_flat and ix.faiss_index.get_param("k_factor") == 4.0
            st = ix.faiss_index.get_state()
            before.append(st)
            o = make_rflat("ivf_pq_fs", d, nlist, M)
            o.set_state(st)
            o.nprobe = 3
            Do, Io = o.search(xq, k)
            Ds.append(Do); Ps.append(Io); metas.append(ix.id_to_metadata)
        Dall = np.stack(Ds)
        pos = np.arange(Dall.size, dtype=np.int64).reshape(Dall.shape)
        refD, refP = O.merge(Dall, pos)
        S_, nq_, k_ = Dall.shape
        want = [[metas[p // (nq_ * k_)][int(Ps[p // (nq_ * k_)][q, p % k_])] for p in refP[q]] for q in range(nq_)]
        for path in ("plane", "sockets"):
            if path == "sockets":
                client.detach_plane()
            D, meta, embs = client.search(xq, k, index_id, return_embeddings=True)
            assert np.array_equal(np.asarray(D, dtype=np.float32), refD), path
            assert [list(r) for r in meta] == want, path
            for q in range(nq_):   # metadata i names row i of everything that was added: the raw rows come back
                for j, m in enumerate(meta[q]):
                    assert np.array_equal(np.asarray(embs[q][j], dtype=np.float32), allx[m]), path
            client.plane = plane
        client.save_index(index_id)
        assert os.path.isfile(os.path.join(store.name, index_id, "0", "index.dfx.npz"))
        client.drop_index(index_id)
        assert client.load_index(index_id, cfg)
        for s, st in zip(servers, before):
            after = s.indexes[index_id].faiss_index.get_state()
            for key in ("centroids", "codebooks", "list_off", "ids", "codes", "refine_vecs", "k_factor"):
                assert np.asarray(after[key]).tobytes() == np.asarray(st[key]).tobytes(), key
        client.set_nprobe(index_id, 3)
        for path in ("plane", "sockets"):
            if path == "sockets":
                client.detach_plane()
            D1, M1 = client.search(xq, k, index_id)
            assert np.array_equal(np.asarray(D1, dtype=np.float32), refD) and [list(r) for r in M1] == want, path
            client.plane = plane
    finally:
        client.close()
        plane.stop()
        for s in servers:
            s.stop()
