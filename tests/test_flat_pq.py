"""Product-quantized flat shards ("PQ{M}", faiss IndexPQ(d, M, 8, metric)) under both metrics.

The canonical answer is the one of tests/oracle_flat_pq.py (DESIGN.md section 2): numpy fp32 tables with a
correctly rounded fmaf, the halving tree, the total order (value, id).  The CPU tests check the parser,
the oracle against float64, the host logic through oracle engines and the persistence; the `gpu` tests
check the engine bit for bit against the oracle over every code width, both scoring paths (the fused
per-tile top-k for k <= 100 or nq * k <= 16384, the values tiles otherwise), training, adds, reconstruction,
range search and the clients."""
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

from distributed_faiss_b200 import faiss_io
from distributed_faiss_b200.factory import ACCEPTED_FORMS, FactorySpec, parse_factory
from distributed_faiss_b200.index import Index, factory_spec
from distributed_faiss_b200.index_cfg import IndexCfg
from tests.conftest import clustered
from tests.oracle_flat_pq import OracleFlatPQ, encode, flat_pq_engine_factory, tables

IP, L2 = 0, 1
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMU = bool(os.environ.get("DFX_EMU_LIB"))
F32 = np.float32


def _sz(full, emu):
    return emu if EMU else full


# ------------------------------------------------------------------ parser
@pytest.mark.parametrize("metric", [IP, L2])
@pytest.mark.parametrize("s", ["PQ16", "PQ16x8"])
def test_parser_maps_pq_to_the_flat_pq_kind(metric, s):
    assert "PQ{M}" in ACCEPTED_FORMS and "PQ{M}x8" in ACCEPTED_FORMS
    assert parse_factory(64, s, metric) == FactorySpec("flat_pq", metric, 0, 16)
    assert factory_spec(IndexCfg(faiss_factory=s, dim=64)) == FactorySpec("flat_pq", IP, 0, 16)  # default: dot
    assert factory_spec(IndexCfg(faiss_factory=s, dim=64, metric="l2")) == FactorySpec("flat_pq", L2, 0, 16)


@pytest.mark.parametrize("d,M,ok", [(64, 4, True), (768, 128, True), (768, 96, True), (96, 12, True),
                                    (64, 6, False), (64, 2, False), (256, 256, False), (132, 132, False),
                                    (100, 8, False), (48, 32, False)])
def test_parser_m_limits(d, M, ok):
    if ok:
        assert parse_factory(d, f"PQ{M}", L2) == FactorySpec("flat_pq", L2, 0, M)
    else:
        with pytest.raises(RuntimeError, match="must be a multiple of 4, at most 128, that divides d"):
            parse_factory(d, f"PQ{M}", L2)


@pytest.mark.parametrize("s", ["PQ16x4", "PQ16x4fs", "PQ16np", "PQ16,RFlat", "OPQ16,PQ16", "PQ16x8,RFlat",
                               "PQ0", "PQ016", "pq16", "PQ16 ", "PQ16x16"])
def test_other_pq_forms_without_lists_stay_rejected(s):
    with pytest.raises(RuntimeError, match="accepted forms"):
        parse_factory(64, s, L2)


def test_ivf_codecs_still_refuse_inner_product_and_ivf_gpu_refuses_pq():
    with pytest.raises(RuntimeError, match="inner-product distance tables"):
        parse_factory(64, "IVF16,PQ16", IP)
    with pytest.raises(RuntimeError, match="needs an IVF factory string"):
        factory_spec(IndexCfg(index_builder_type="ivf_gpu", faiss_factory="PQ16", dim=64))


# ------------------------------------------------------------------ oracle
def _trained_oracle(rs, d, M, metric, n):
    o = OracleFlatPQ(d, M, metric)
    o.codebooks = rs.randn(M, 256, d // M).astype(F32)
    o.is_trained = True
    o.add(rs.randn(n, d).astype(F32))
    return o


@pytest.mark.parametrize("metric", [IP, L2])
@pytest.mark.parametrize("d,M", [(48, 12), (64, 16), (160, 80)])
def test_oracle_against_a_float64_restatement(metric, d, M, oracle_lib):
    rs = np.random.RandomState(3 + M)
    n, k = 600, 20
    o = _trained_oracle(rs, d, M, metric, n)
    xq = rs.randn(9, d).astype(F32)
    D, I = o.search(xq, k)
    xhat = o.reconstruct_rows(np.arange(n)).astype(np.float64)
    q = xq.astype(np.float64)
    ref = ((q[:, None, :] - xhat[None]) ** 2).sum(-1) if metric == L2 else -(q @ xhat.T)
    got = D.astype(np.float64) if metric == L2 else -D.astype(np.float64)
    want = np.take_along_axis(ref, I, 1)
    slack = 1e-5 * (np.abs(ref).max() + 1)                       # fp32 rounding of M table sums
    assert np.all(np.abs(got - want) <= slack)
    order = np.argsort(ref, axis=1, kind="stable")[:, :k]
    sep = np.diff(np.sort(ref, axis=1)[:, :k + 1], axis=1).min(axis=1) > 4 * slack
    assert sep.any()
    assert np.array_equal(I[sep], order[sep])
    assert np.array_equal(encode(o.codebooks, xhat.astype(F32)), o.codes)   # a codeword encodes to itself


def test_tables_follow_the_canonical_order(oracle_lib):
    rs = np.random.RandomState(4)
    cb = rs.randn(4, 256, 3).astype(F32)
    x = rs.randn(2, 12).astype(F32)
    l2, ip = tables(cb, x, L2), tables(cb, x, IP)
    for q in range(2):
        for m in range(4):
            for j in (0, 77, 255):
                a = F32(0)
                b = F32(0)
                for t in range(3):
                    df = F32(x[q, 3 * m + t] - cb[m, j, t])
                    a = F32(np.float64(df) * np.float64(df) + np.float64(a))
                    b = F32(np.float64(x[q, 3 * m + t]) * np.float64(cb[m, j, t]) + np.float64(b))
                assert l2[q, m, j] == a and ip[q, m, j] == -b


# ------------------------------------------------------------------ persistence
def _state(metric, n=57, d=24, M=8, seed=4):
    o = _trained_oracle(np.random.RandomState(seed), d, M, metric, n)
    return o, o.get_state()


@pytest.mark.parametrize("metric", [IP, L2])
def test_ixpq_byte_layout_round_trip(metric, tmp_path, oracle_lib):
    o, st = _state(metric)
    assert st["kind"] == "flat_pq" and st["metric"] == metric and st["M"] == 8 and st["ksub"] == 256
    path = str(tmp_path / "ix.faiss")
    faiss_io.write_index(st, path)
    raw = open(path, "rb").read()
    n, M = st["codes"].shape
    d = st["d"]
    want = b"IxPq" + struct.pack("<iqqqBi", d, n, 1 << 20, 1 << 20, 1, metric)
    want += struct.pack("<QQQ", d, M, 8) + struct.pack("<Q", M * 256 * (d // M)) + st["codebooks"].astype("<f4").tobytes()
    want += struct.pack("<Q", n * M) + st["codes"].tobytes() + struct.pack("<iBi", 0, 0, 0)
    assert raw == want
    back, nprobe = faiss_io.read_index(path)
    assert back["kind"] == "flat_pq" and back["metric"] == metric and back["d"] == d and back["M"] == M
    assert np.array_equal(back["codes"], st["codes"]) and np.array_equal(back["codebooks"], st["codebooks"])
    o2 = OracleFlatPQ(d, M, metric)
    o2.set_state(back)
    q = np.random.RandomState(0).randn(5, d).astype(F32)
    assert all(a.tobytes() == b.tobytes() for a, b in zip(o.search(q, 6), o2.search(q, 6)))


def test_ixpq_refuses_polysemous_search_and_other_nbits(tmp_path, oracle_lib):
    _, st = _state(L2, n=4)
    path = str(tmp_path / "ix.faiss")
    faiss_io.write_index(st, path)
    raw = bytearray(open(path, "rb").read())
    bad = bytearray(raw)
    bad[-9:-5] = struct.pack("<i", 1)                              # search_type ST_HE
    with pytest.raises(faiss_io.FaissFormatError, match="search_type"):
        faiss_io.read_index(_write(tmp_path, bad))
    off = 4 + struct.calcsize("<iqqqBi") + 16
    bad = bytearray(raw)
    bad[off:off + 8] = struct.pack("<Q", 4)                        # nbits = 4
    with pytest.raises(faiss_io.FaissFormatError, match="8 bits"):
        faiss_io.read_index(_write(tmp_path, bad))


def _write(tmp_path, raw):
    p = str(tmp_path / "bad.faiss")
    open(p, "wb").write(bytes(raw))
    return p


def _wait_added(ix):
    import time

    from distributed_faiss_b200.index_state import IndexState

    t0 = time.time()
    while ix.get_state() != IndexState.TRAINED:
        assert time.time() - t0 < 120
        time.sleep(0.02)


def _drop_stored_cfg(storage_dir):
    from distributed_faiss_b200.index import get_index_files

    os.remove(get_index_files(storage_dir)[3])


@pytest.mark.parametrize("fmt", ["dfx", "faiss"])
@pytest.mark.parametrize("metric", ["dot", "l2"])
def test_save_load_and_kind_mismatch_refusals(fmt, metric, oracle_lib):
    rs = np.random.RandomState(6)
    d = 16
    with tempfile.TemporaryDirectory() as tmp:
        cfg = IndexCfg(faiss_factory="PQ4", dim=d, metric=metric, index_storage_dir=tmp, index_format=fmt,
                       train_num=300)
        ix = Index(cfg, engine_factory=flat_pq_engine_factory)
        x = rs.randn(400, d).astype(F32)
        ix.add_batch(x, list(range(400)), train_async_if_triggered=False)
        _wait_added(ix)
        assert isinstance(ix.faiss_index, OracleFlatPQ) and ix.faiss_index.ntotal == 400
        D0, M0, _ = ix.search(x[:7], 5)
        ix.save()
        back = Index.from_storage_dir(tmp, cfg, engine_factory=flat_pq_engine_factory)
        assert isinstance(back.faiss_index, OracleFlatPQ)
        assert np.array_equal(back.faiss_index.codes, ix.faiss_index.codes)
        D1, M1, _ = back.search(x[:7], 5)
        assert np.array_equal(D0, D1) and M0 == M1
        _drop_stored_cfg(tmp)
        # another M, and another kind (fp32 flat) under the same stored shard
        other_m = IndexCfg(faiss_factory="PQ8", dim=d, metric=metric, index_storage_dir=tmp, index_format=fmt)
        with pytest.raises(RuntimeError, match=r"the stored PQ index has \(M, ksub\) = \(4, 256\).*refusing"):
            Index.from_storage_dir(tmp, other_m, engine_factory=flat_pq_engine_factory)
        flat_cfg = IndexCfg(faiss_factory="Flat", dim=d, metric=metric, index_storage_dir=tmp, index_format=fmt)
        with pytest.raises(RuntimeError, match="refusing to load it"):
            Index.from_storage_dir(tmp, flat_cfg, engine_factory=flat_pq_engine_factory)
    with tempfile.TemporaryDirectory() as tmp:
        flat_cfg = IndexCfg(faiss_factory="Flat", dim=d, metric=metric, index_storage_dir=tmp, index_format=fmt,
                            train_num=10)
        ix = Index(flat_cfg, engine_factory=flat_pq_engine_factory)
        ix.add_batch(rs.randn(50, d).astype(F32), list(range(50)), train_async_if_triggered=False)
        _wait_added(ix)
        ix.save()
        _drop_stored_cfg(tmp)
        pq_cfg = IndexCfg(faiss_factory="PQ4", dim=d, metric=metric, index_storage_dir=tmp, index_format=fmt)
        with pytest.raises(RuntimeError, match="refusing to load it"):
            Index.from_storage_dir(tmp, pq_cfg, engine_factory=flat_pq_engine_factory)


# ------------------------------------------------------------------ host logic through oracle engines
@pytest.fixture(scope="module")
def servers():
    from distributed_faiss_b200.client import ResultHeap
    from distributed_faiss_b200.server import IndexServer
    from tests.oracle_engine import oracle_merge
    from tests.test_host_logic import free_ports, wait_listening

    ResultHeap.merge_backend = staticmethod(oracle_merge)
    store = tempfile.TemporaryDirectory()
    ports = free_ports(2)
    srv = []
    for i, p in enumerate(ports):
        s = IndexServer(i, store.name, engine_factory=flat_pq_engine_factory)
        threading.Thread(target=s.start_blocking, args=(p,), daemon=True).start()
        srv.append(s)
    wait_listening(ports)
    yield ports, srv
    for s in srv:
        s.stop()


@pytest.mark.parametrize("metric", ["dot", "l2"])
def test_sharded_search_through_servers_with_oracle_engines(servers, metric, oracle_lib):
    """two shards behind IndexServers: the client's merged D and metadata equal the merge of the shards'
    own answers (the client negates for dot, as for every kind), with and without return_embeddings"""
    from oracle import oracle as O
    from tests.test_host_logic import make_client, wait_trained

    ports, srv = servers
    rs = np.random.RandomState(7)
    d, index_id = 32, f"pq_{metric}"
    client = make_client(ports)
    client.create_index(index_id, IndexCfg(faiss_factory="PQ8", dim=d, metric=metric, train_num=260))
    for b in range(4):
        client.add_index_data(index_id, clustered(rs, 300, d, ncl=8), [(b, i) for i in range(300)], False)
    client.sync_train(index_id)
    wait_trained(client, index_id)
    shards = [s.indexes[index_id] for s in srv]
    assert all(isinstance(ix.faiss_index, OracleFlatPQ) and ix.faiss_index.metric == (IP if metric == "dot" else L2)
               for ix in shards)
    q = clustered(rs, 9, d, ncl=8)
    per = [ix.faiss_index.search(q, 10) for ix in shards]
    Dall = np.stack([D for D, _ in per])
    pos = np.arange(Dall.size, dtype=np.int64).reshape(Dall.shape)
    neg = metric == "dot"
    Dref, P = O.merge(-Dall if neg else Dall, pos)
    meta = [ix.id_to_metadata[i] if i >= 0 else None for ix, (_, I) in zip(shards, per) for i in I.reshape(-1)]
    rows = np.concatenate([ix.faiss_index.reconstruct_rows(I.reshape(-1)) for ix, (_, I) in zip(shards, per)])
    Dm, Mm = client.search(q, 10, index_id)
    assert np.array_equal(Dm, Dref) and Mm == [[meta[p] if p >= 0 else None for p in row] for row in P]
    Dm, Mm, Em = client.search(q, 10, index_id, True)
    assert np.array_equal(Dm, Dref)
    assert np.array_equal(np.asarray(Em).reshape(-1, d), rows[P.reshape(-1)])
    client.close()


# ------------------------------------------------------------------ on the emulated library
EMU_SUBSET = [
    "tests/test_flat_pq.py::test_search_matches_the_oracle[0-64-8-2049]",
    "tests/test_flat_pq.py::test_search_matches_the_oracle[1-96-12-300]",
    "tests/test_flat_pq.py::test_search_matches_the_oracle[1-160-80-2048]",
    "tests/test_flat_pq.py::test_search_matches_the_oracle[0-128-128-700]",
    "tests/test_flat_pq.py::test_training_and_encoding_match_the_restatement[64-16]",
    "tests/test_flat_pq.py::test_adds_in_batches_reconstruct_and_index_bytes",
    "tests/test_flat_pq.py::test_range_search_is_the_cut_knn_search",
    "tests/test_flat_pq.py::test_refusals",
]


def test_gpu_subset_on_the_emulated_library():
    if EMU:
        pytest.skip("already running on the emulated library")
    if shutil.which("g++") is None or platform.machine() != "x86_64":
        pytest.skip("the emulator needs g++ on x86-64")
    sys.path.insert(0, os.path.join(ROOT, "tests", "emu"))
    try:
        import build_emu_lib
    finally:
        sys.path.pop(0)
    env = dict(os.environ, DFX_EMU_LIB=build_emu_lib.build())
    run = subprocess.run([sys.executable, "-m", "pytest", "-m", "gpu", "-q", "-x", "-p", "no:cacheprovider"] + EMU_SUBSET,
                         cwd=ROOT, env=env, capture_output=True, text=True, timeout=2400)
    tail = (run.stdout + run.stderr)[-3000:]
    assert run.returncode == 0, tail
    assert f"{len(EMU_SUBSET)} passed" in run.stdout, tail


# ------------------------------------------------------------------ GPU: the engine
def _engine():
    from distributed_faiss_b200 import engine

    return engine


def _same(a, b, what):
    (Da, Ia), (Db, Ib) = a, b
    assert Da.shape == Db.shape, (what, Da.shape, Db.shape)
    if not (np.array_equal(Ia, Ib) and np.array_equal(Da.view(np.uint32), Db.view(np.uint32))):
        bad = np.argwhere((Ia != Ib) | (Da.view(np.uint32) != Db.view(np.uint32)))
        q, j = bad[0]
        raise AssertionError(f"{what}: {len(bad)} slots differ; first q={q} j={j}: ({Da[q, j]!r},{Ia[q, j]}) vs "
                             f"({Db[q, j]!r},{Ib[q, j]})")


def _shard(d, M, metric, x, xt=None, niter=2):
    """a trained FLAT_PQ shard holding x (trained on xt, default x), and its oracle from the shard's state"""
    E = _engine()
    g = E.GpuIndex(E.KIND_FLAT_PQ, d, metric, pq_m=M)
    g.set_param("kmeans_niter", niter)
    g.train(x if xt is None else xt)
    if len(x):
        g.add(x)
    o = OracleFlatPQ(d, M, metric)
    o.set_state(g.get_state())
    return g, o


def _data(rs, n, d):
    x = clustered(rs, max(n, 1), d, ncl=max(8, n // 400))[:n] * F32(3)
    m = n // 20
    if m:
        x[n - m:] = x[:m]                                        # exact duplicates: ties broken by id
    return x


# (metric, d, M, N): every code width (8, 16, 32, 64, 96, 128 and the generic narrow / wide shapes), N = 0,
# N < k, one tile, a fused tile boundary +-1 (2048-row tiles at small batches), a values tile boundary +-1
# (32768), several tiles
SHAPES = [(0, 64, 8, 2049), (1, 64, 16, 0), (0, 64, 16, 100), (1, 128, 32, 2047), (0, 128, 64, 32769),
          (1, 128, 64, 32767), (0, 128, 128, 700), (1, 768, 96, 3000), (0, 768, 64, 6000), (1, 768, 128, 2048),
          (1, 96, 12, 300), (0, 96, 12, 4097), (1, 160, 80, 2048), (1, 64, 32, 70000)]


@pytest.mark.gpu
@pytest.mark.parametrize("metric,d,M,N", SHAPES, ids=[f"{m}-{d}-{M}-{n}" for m, d, M, n in SHAPES])
def test_search_matches_the_oracle(metric, d, M, N):
    rs = np.random.RandomState(d + M + N + metric)
    xt = _data(rs, 600, d)
    x = _data(rs, N, d)
    g, o = _shard(d, M, metric, x, xt)
    # the first and last 1024 codes (the training test checks the encode of every row)
    rows = np.unique(np.r_[np.arange(min(N, 1024)), np.arange(max(0, N - 1024), N)])
    assert g.ntotal == N and np.array_equal(g.get_array("codes").reshape(-1, M)[rows], encode(o.codebooks, x[rows]))
    xq = np.concatenate([x[:: max(1, N // 500)][:500], clustered(rs, 600, d, ncl=8)])
    ks = (1, 32, 33, 1024, 1025, 4096) if not EMU else (1, 33, 1025)
    nqs = ((1, 7, 1025) if N <= 6000 and d <= 128 else (1, 7)) if not EMU else (1, 7)
    for nq in nqs:
        q = xq[:nq]
        want = o.search(q, max(ks))
        for k in ks:
            _same(g.search(q, k), (want[0][:, :k], want[1][:, :k]), f"N={N} nq={nq} k={k}")


# (nq, k) that take the fused per-tile top-k (k <= 100, or nq * k <= 16384; DESIGN.md section 4.14); k = 1025
# takes the values tiles
FUSED_CASES = ((1, 1024), (16, 1024), (64, 256), (1025, 100), (1025, 10))


@pytest.mark.gpu
@pytest.mark.parametrize("metric", [IP, L2])
def test_fused_and_values_paths_agree(metric):
    """the fused per-tile top-k at k is the first k columns of the values tiles at k = 1025"""
    rs = np.random.RandomState(30 + metric)
    d, M, N = 128, 32, _sz(100_000, 3000)
    x = _data(rs, N, d)
    g, _ = _shard(d, M, metric, x, x[:2000])
    for nq, k in FUSED_CASES if not EMU else ((1, 1024), (3, 100)):
        q = x[:nq] + F32(0.01)
        D1, I1 = g.search(q, 1025)
        _same(g.search(q, k), (D1[:, :k], I1[:, :k]), f"nq={nq} k={k}")


@pytest.mark.gpu
def test_fused_path_under_its_query_chunk_cap():
    """N = 5.6 M rows: at k = 100 the 1025 queries' partial rows (171 tiles of 32768 rows x 100 composites
    each) would exceed the 2^24 composites of a chunk, so the fused path runs two chunks (981 + 44 queries);
    the answer is the first 100 columns of the values tiles at k = 1025"""
    import torch

    E = _engine()
    d, M, N, k = 32, 8, 5_600_000, 100
    gen = torch.Generator(device="cuda").manual_seed(36)
    x = torch.randn(N, d, device="cuda", generator=gen)
    part_max, tile = 1 << 24, 32768
    assert part_max // ((-(-N // tile)) * k) < 1024               # the cap binds
    for metric in (IP, L2):
        g = E.GpuIndex(E.KIND_FLAT_PQ, d, metric, pq_m=M)
        g.set_param("kmeans_niter", 2)
        g.train_dev(x[:4096].contiguous())
        g.add_dev(x)
        q = (x[:1025] + 0.01).contiguous()
        D, I = g.search_dev(q, k)
        D1, I1 = g.search_dev(q, 1025)
        _same((D.cpu().numpy(), I.cpu().numpy()), (D1[:, :k].cpu().numpy(), I1[:, :k].cpu().numpy()),
              f"metric={metric} chunk cap")
        del g


@pytest.mark.gpu
@pytest.mark.parametrize("d,M", [(64, 16), (48, 16), (768, 128)])
def test_training_and_encoding_match_the_restatement(d, M):
    """the codebooks are the device k-means of tests/oracle_train on the first rows, the codes the oracle's
    (dsub 4: the register encode, dsub 3 and 6: the generic one)"""
    rs = np.random.RandomState(31 + d)
    x = clustered(rs, _sz(1500, 400), d, ncl=32)
    E = _engine()
    g = E.GpuIndex(E.KIND_FLAT_PQ, d, L2, pq_m=M)
    g.set_param("kmeans_niter", 2)
    g.train(x)
    o = OracleFlatPQ(d, M, L2)
    o.train_niter = 2
    o.train(x)
    got = g.get_array("codebooks").reshape(M, 256, d // M)
    bad = np.argwhere(got.view(np.uint32) != o.codebooks.view(np.uint32))
    assert not len(bad), f"{len(bad)} codebook values differ, first at {tuple(bad[0])}"
    g.add(x)
    assert np.array_equal(g.get_array("codes").reshape(-1, M), encode(o.codebooks, x))


@pytest.mark.gpu
def test_adds_in_batches_reconstruct_and_index_bytes():
    rs = np.random.RandomState(32)
    d, M = 64, 16
    x = _data(rs, _sz(5000, 2100), d)
    q = x[:9] + F32(0.01)
    for metric in (IP, L2):
        g1, o = _shard(d, M, metric, x, x[:800])
        E = _engine()
        g3 = E.GpuIndex(E.KIND_FLAT_PQ, d, metric, pq_m=M)
        g3.set_state({k: v for k, v in g1.get_state().items() if k != "codes"} | {"codes": np.zeros((0, M), np.uint8)})
        cuts = [0, 700, 701, 2100, len(x)]
        for a, b in zip(cuts[:-1], cuts[1:]):                      # searches between the adds
            g3.add(x[a:b])
            _same(g3.search(q, 10), OracleFlatPQ.search(_prefix(o, b), q, 10), f"metric={metric} after {b}")
        _same(g3.search(q, 50), g1.search(q, 50), f"metric={metric} batches")
        ids = np.array([0, 5, len(x) - 1, -1, len(x)])
        R = g3.reconstruct_rows(ids)
        assert np.array_equal(R[:3], o.reconstruct_rows(ids[:3])) and np.isnan(R[3:]).all()
        D, I, R = g1.search_and_reconstruct(q, 10)
        _same((D, I), o.search(q, 10), f"search_and_reconstruct metric={metric}")
        assert np.array_equal(R.reshape(-1, d), o.reconstruct_rows(I.reshape(-1)))
        # N M bytes of codes plus the codebooks (M x 256 x d / M floats): 1 + 4 d N^-1 ... per vector
        assert g1.get_param("index_bytes") == len(x) * M + 256 * d * 4


def _prefix(o, n):
    p = OracleFlatPQ(o.d, o.M, o.metric)
    p.codebooks, p.codes, p.is_trained = o.codebooks, o.codes[:n], True
    return p


@pytest.mark.gpu
def test_range_search_is_the_cut_knn_search():
    """every (D, I) pair of a range search is the pair search at k = 4096 reports, cut at the radius
    (strict, faiss's direction per metric), +-inf radii included"""
    rs = np.random.RandomState(33)
    d, M = 64, 16
    for metric in (IP, L2):
        for N in (3000,) if EMU else (3000, 40000):
            x = _data(rs, N, d)
            g, _ = _shard(d, M, metric, x, x[:800])
            q = x[:13] + F32(0.01)
            D, I = g.search(q, 4096)
            radii = [float(np.median(D[:, 20]))]
            if N <= 4096:
                radii += [np.inf, -np.inf]
            for r in radii:
                lims, Dr, Ir = g.range_search(q, r)
                for i in range(len(q)):
                    keep = (D[i] < r) if metric == L2 else (D[i] > r)
                    keep &= I[i] >= 0
                    assert np.array_equal(Ir[lims[i]:lims[i + 1]], I[i][keep]), (metric, N, r, i)
                    assert np.array_equal(Dr[lims[i]:lims[i + 1]].view(np.uint32), D[i][keep].view(np.uint32))


@pytest.mark.gpu
def test_refusals():
    E = _engine()
    for kw, msg in ((dict(pq_m=6), "multiple of 4, at most 128, that divides d"),
                    (dict(pq_m=256), "multiple of 4, at most 128, that divides d"),
                    (dict(pq_m=16, pq_nbits=4), "8 bits per sub-quantizer"),
                    (dict(pq_m=16, nlist=4), "must be 0")):
        with pytest.raises(RuntimeError, match=msg):
            E.GpuIndex(E.KIND_FLAT_PQ, 64, L2, **kw)
    g = E.GpuIndex(E.KIND_FLAT_PQ, 64, IP, pq_m=16)
    assert not g.is_trained and g.nlist == 0 and g.search_metric == IP
    x = np.random.RandomState(34).randn(300, 64).astype(F32)
    with pytest.raises(RuntimeError, match="not trained"):
        g.search(x[:2], 5)
    with pytest.raises(RuntimeError, match="not trained"):
        g.add(x)
    with pytest.raises(RuntimeError, match="need at least 256 vectors for PQ"):
        g.train(x[:255])
    g.set_param("kmeans_niter", 1)
    g.train(x)
    assert g.is_trained and g.ntotal == 0
    D, I = g.search(x[:2], 5)                                    # N = 0: padding only
    assert (I == -1).all() and (D == -np.finfo(F32).max).all()


@pytest.mark.gpu
def test_client_over_sockets_and_the_search_plane():
    from distributed_faiss_b200.index_cfg import IndexCfg as Cfg
    from oracle import oracle as O
    from tests.test_gpu_api import _both_ways, _plane_cluster, wait_trained

    store, servers, plane, client = _plane_cluster(2)
    rs = np.random.RandomState(35)
    d = 128
    try:
        for metric in ("dot", "l2"):
            name = f"pq_{metric}"
            client.create_index(name, Cfg(faiss_factory="PQ32", dim=d, metric=metric, train_num=1000))
            for b in range(4):
                client.add_index_data(name, clustered(rs, 1500, d, ncl=16), [(b, i) for i in range(1500)], False)
            client.sync_train(name)
            wait_trained(client, name)
            shards = [s.indexes[name] for s in servers]
            assert all(ix.faiss_index.kind == _engine().KIND_FLAT_PQ for ix in shards)
            q = clustered(rs, 40, d, ncl=16)
            per = [ix.faiss_index.search(q, 10) for ix in shards]
            Dall = np.stack([D for D, _ in per])
            pos = np.arange(Dall.size, dtype=np.int64).reshape(Dall.shape)
            Dref, P = O.merge(-Dall if metric == "dot" else Dall, pos)
            meta = [ix.id_to_metadata[i] if i >= 0 else None for ix, (_, I) in zip(shards, per) for i in I.reshape(-1)]
            rows = np.concatenate([ix.faiss_index.reconstruct_rows(I.reshape(-1)) for ix, (_, I) in zip(shards, per)])
            Mref = [[meta[p] if p >= 0 else None for p in row] for row in P]
            (Dp, Mp), (Ds, Ms) = _both_ways(client, plane, lambda: client.search(q, 10, name))
            for D, M in ((Dp, Mp), (Ds, Ms)):
                assert np.array_equal(D, Dref) and list(M) == Mref
            (Dp, Mp, Ep), (Ds, Ms, Es) = _both_ways(client, plane, lambda: client.search(q, 10, name, True))
            for D, M, E in ((Dp, Mp, Ep), (Ds, Ms, Es)):
                assert np.array_equal(D, Dref) and list(M) == Mref
                assert np.array_equal(np.asarray(E).reshape(-1, d), rows[P.reshape(-1)])
    finally:
        client.close()
        plane.stop()
        for s in servers:
            s.stop()
