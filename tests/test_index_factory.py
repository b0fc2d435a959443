"""faiss_factory strings and the ivf_gpu builder (reference index.py:71-86, 385-396): the parser,
and the host logic (sharding, nprobe rules, persistence) through oracle engines built by the same
parser (tests/oracle_sq8.oracle_engine_factory)."""
import os
import tempfile
import threading

import numpy as np
import pytest

from distributed_faiss_b200.client import ResultHeap
from distributed_faiss_b200.factory import ACCEPTED_FORMS, FactorySpec, parse_factory, substitute_centroids
from distributed_faiss_b200.index import Index, factory_spec
from distributed_faiss_b200.index_cfg import IndexCfg
from distributed_faiss_b200.index_state import IndexState
from distributed_faiss_b200.server import IndexServer
from tests.conftest import clustered
from tests.oracle_engine import oracle_merge
from tests.oracle_sq8 import OracleIVFSQ8, oracle_engine_factory
from tests.test_host_logic import free_ports, make_client, wait_listening, wait_trained

IP, L2 = 0, 1


# ------------------------------------------------------------------ parser
@pytest.mark.parametrize("s,metric,want", [
    ("Flat", IP, FactorySpec("flat", IP)),
    ("Flat", L2, FactorySpec("flat", L2)),
    ("IVF64,Flat", IP, FactorySpec("ivf_flat", IP, 64)),
    ("IVF64,Flat", L2, FactorySpec("ivf_flat", L2, 64)),
    ("IVF100,PQ16", L2, FactorySpec("ivf_pq", L2, 100, 16)),
    ("IVF100,PQ16x8", L2, FactorySpec("ivf_pq", L2, 100, 16)),
    ("IVF7,SQfp16", L2, FactorySpec("ivf_sq", L2, 7)),
    ("IVF4096,SQ8", L2, FactorySpec("ivf_sq8", L2, 4096)),
])
def test_accepted_forms(s, metric, want):
    assert parse_factory(64, s, metric) == want


@pytest.mark.parametrize("s", [
    "OPQ16,IVF64,PQ16", "PCA32,IVF64,Flat", "HNSW32", "HNSW32,SQ8", "IVF64_HNSW32,Flat", "IVF64,Flat,RFlat",
    "IVF64,PQ16,Refine(Flat)", "IDMap,Flat", "IVF64,PQ16x4", "IVF64,SQ4", "IVF64,SQ6", "IVF,Flat", "IVF0,Flat",
    "IVF064,Flat", "IVFx,SQ8", "IVF{centroids},SQ8", "IVF64,PQ", "IVF64,PQ0", "ivf64,flat", "flat", "IVF64,sq8",
    "IVF64, SQ8", "", "SQ8", "IVF64,SQ8,", "LSH",
])
def test_rejected_forms_name_the_string_and_the_accepted_ones(s):
    with pytest.raises(RuntimeError) as e:
        parse_factory(64, s, L2)
    assert repr(s) in str(e.value) and all(f in str(e.value) for f in ACCEPTED_FORMS)


@pytest.mark.parametrize("s", ["IVF64,PQ16", "IVF64,PQ16x8", "IVF64,SQfp16", "IVF64,SQ8"])
def test_inner_product_with_a_codec_has_its_own_message(s):
    with pytest.raises(RuntimeError, match="inner-product distance tables"):
        parse_factory(64, s, IP)


@pytest.mark.parametrize("s", ["IVF64,PQ6", "IVF64,PQ128", "IVF64,PQ12"])   # not %4, > 64, 64 % 12 != 0
def test_pq_sub_quantizer_limits(s):
    with pytest.raises(RuntimeError, match="sub-quantizers"):
        parse_factory(64, s, L2)


def test_factory_path_and_ivf_gpu_rules():
    # factory path (index.py:385-396): {centroids} substituted, cfg metric, nlist from the string
    cfg = IndexCfg(faiss_factory="IVF{centroids},SQ8", dim=32, centroids=12, metric="l2", nprobe=5)
    assert substitute_centroids(cfg.faiss_factory, 12) == "IVF12,SQ8"
    assert factory_spec(cfg) == FactorySpec("ivf_sq8", L2, 12)
    cfg = IndexCfg(faiss_factory="IVF9,Flat", dim=32, centroids=12, metric="dot")
    assert factory_spec(cfg) == FactorySpec("ivf_flat", IP, 9)
    with pytest.raises(RuntimeError, match="inner-product"):
        factory_spec(IndexCfg(faiss_factory="IVF{centroids},SQ8", dim=32, centroids=4, metric="dot"))
    # ivf_gpu (index.py:71-86): raw string, always L2
    cfg = IndexCfg(index_builder_type="ivf_gpu", faiss_factory="IVF16,SQ8", dim=32, metric="dot", nprobe=3)
    assert factory_spec(cfg) == FactorySpec("ivf_sq8", L2, 16)
    cfg = IndexCfg(index_builder_type="ivf_gpu", faiss_factory="IVF16,Flat", dim=32, metric="dot")
    assert factory_spec(cfg) == FactorySpec("ivf_flat", L2, 16)
    with pytest.raises(RuntimeError, match="not supported"):   # no substitution on this path
        factory_spec(IndexCfg(index_builder_type="ivf_gpu", faiss_factory="IVF{centroids},SQ8", dim=32, centroids=4))
    with pytest.raises(RuntimeError, match="IVF factory string"):
        factory_spec(IndexCfg(index_builder_type="ivf_gpu", faiss_factory="Flat", dim=32))
    # a builder name wins over a factory string, as in the reference
    assert factory_spec(IndexCfg(index_builder_type="ivfsq", faiss_factory="IVF4,SQ8", dim=32)) is None


def test_oracle_engines_follow_the_nprobe_rules():
    ix = oracle_engine_factory(IndexCfg(faiss_factory="IVF{centroids},SQ8", dim=16, centroids=8, metric="l2", nprobe=5))
    assert isinstance(ix, OracleIVFSQ8) and ix.nlist == 8 and ix.nprobe == 1      # faiss default
    cfg = IndexCfg(index_builder_type="ivf_gpu", faiss_factory="IVF8,SQ8", dim=16, metric="dot", nprobe=5)
    ix = oracle_engine_factory(cfg)
    assert isinstance(ix, OracleIVFSQ8) and ix.nprobe == 5 and ix.coarse_metric == L2 and cfg.nprobe == 5
    ix = oracle_engine_factory(IndexCfg(faiss_factory="Flat", dim=16, metric="l2"))
    assert ix.kind == "flat" and ix.metric == L2                                  # unlike the "flat" builder
    with pytest.raises(RuntimeError):
        oracle_engine_factory(IndexCfg(index_builder_type="hnswsq", dim=16, metric="l2"))


def test_index_infers_centroids_on_the_factory_path():
    cfg = IndexCfg(faiss_factory="IVF{centroids},SQ8", dim=16, centroids=0, metric="l2", nprobe=3, train_num=400)
    ix = Index(cfg, engine_factory=oracle_engine_factory)
    rs = np.random.RandomState(0)
    ix.add_batch(clustered(rs, 400, 16, ncl=8), list(range(400)), train_async_if_triggered=False)
    assert cfg.centroids == int(2 * np.sqrt(400))                                  # index.py:497-508
    assert ix.faiss_index.nlist == cfg.centroids and ix.faiss_index.nprobe == 1 and cfg.nprobe == 3


# ------------------------------------------------------------------ through the servers
@pytest.fixture(scope="module")
def servers():
    ResultHeap.merge_backend = staticmethod(oracle_merge)
    dirs = [tempfile.TemporaryDirectory(), tempfile.TemporaryDirectory()]
    ports = free_ports(4)
    srv = []
    for i, p in enumerate(ports):
        s = IndexServer(i if i < 3 else 0, dirs[0].name if i < 3 else dirs[1].name,
                        engine_factory=oracle_engine_factory)
        threading.Thread(target=s.start_blocking, args=(p,), daemon=True).start()
        srv.append(s)
    wait_listening(ports)
    yield {"multi": ports[:3], "single": ports[3:], "servers": srv, "dirs": dirs}
    for s in srv:
        s.stop()


def _wait_ntotal(client, index_id, n):
    import time

    t0 = time.time()
    while client.get_ntotal(index_id) != n or client.get_state(index_id) != IndexState.TRAINED:
        assert time.time() - t0 < 60
        time.sleep(0.05)


@pytest.mark.parametrize("builder,factory,metric", [
    ("", "IVF{centroids},SQ8", "l2"),
    ("ivf_gpu", "IVF8,SQ8", "l2"),
    ("ivf_gpu", "IVF8,SQ8", "dot"),       # the index is L2, the client still negates (quirk B2)
])
def test_sharded_search_and_nprobe_rules(servers, builder, factory, metric):
    """Every shard trains its own quantizer, so a sharded IVF index is compared with the exact merge
    of its shards' own answers (what one unsharded heap over the same shards returns)."""
    from oracle import oracle as O

    rs = np.random.RandomState(1)
    d = 32
    index_id = f"f_{builder or 'factory'}_{metric}"
    cfg = IndexCfg(index_builder_type=builder or None, faiss_factory=factory, dim=d, centroids=8, metric=metric,
                   nprobe=3)
    multi = make_client(servers["multi"])
    multi.create_index(index_id, cfg)
    xs = []
    for b in range(6):                                   # two batches per shard
        x = clustered(rs, 300, d, ncl=8)
        multi.add_index_data(index_id, x, [(b, i) for i in range(300)], False)
        xs.append(x)
    multi.sync_train(index_id)
    _wait_ntotal(multi, index_id, 1800)
    shards = [s.indexes[index_id] for s in servers["servers"][:3]]
    want_nprobe = 3 if builder == "ivf_gpu" else 1
    for ix in shards:
        assert ix.faiss_index.nprobe == want_nprobe
        assert ix.cfg.nprobe == 3                                     # never overwritten (unlike knnlm)
        assert ix.faiss_index.coarse_metric == L2 and ix.faiss_index.nlist == 8
    q = np.concatenate(xs)[::97][:12] + np.float32(0.01)
    for nprobe in (None, 5):
        if nprobe:
            multi.set_nprobe(index_id, nprobe)
            assert all(ix.faiss_index.nprobe == 5 for ix in shards)
        Dm, Mm = multi.search(q, 10, index_id)
        per = [ix.faiss_index.search(q, 10) for ix in shards]
        Dall = np.stack([D for D, _ in per])
        pos = np.arange(Dall.size, dtype=np.int64).reshape(Dall.shape)
        neg = metric == "dot"
        Dref, P = O.merge(-Dall if neg else Dall, pos)
        meta = [ix.id_to_metadata[i] if i >= 0 else None for ix, (_, I) in zip(shards, per) for i in I.reshape(-1)]
        assert np.array_equal(Dm, Dref)
        assert Mm == [[meta[p] if p >= 0 else None for p in row] for row in P]
        if neg:
            assert (Dm <= 0).all() and (np.diff(Dm, axis=1) >= 0).all()
    multi.close()


@pytest.mark.parametrize("fmt", ["dfx", "faiss"])
def test_factory_shards_save_and_load(servers, fmt):
    rs = np.random.RandomState(2)
    d = 32
    index_id = f"f_save_{fmt}"
    cfg = IndexCfg(faiss_factory="IVF{centroids},SQ8", dim=d, centroids=8, metric="l2", nprobe=4, index_format=fmt)
    client = make_client(servers["single"])
    client.create_index(index_id, cfg)
    x = clustered(rs, 700, d, ncl=8)
    client.add_index_data(index_id, x, list(range(700)), False)
    client.sync_train(index_id)
    _wait_ntotal(client, index_id, 700)
    client.set_nprobe(index_id, 4)
    D0, M0 = client.search(x[:9], 7, index_id)
    client.save_index(index_id)
    shard_dir = os.path.join(servers["dirs"][1].name, index_id, "0")
    assert os.path.isfile(os.path.join(shard_dir, "index.faiss" if fmt == "faiss" else "index.dfx.npz"))
    before = servers["servers"][3].indexes[index_id].faiss_index.get_state()
    client.drop_index(index_id)
    client.close()
    c2 = make_client(servers["single"])
    assert c2.load_index(index_id, cfg)                               # a load with a cfg applies cfg.nprobe
    ix = servers["servers"][3].indexes[index_id]
    assert isinstance(ix.faiss_index, OracleIVFSQ8) and ix.faiss_index.nprobe == 4
    after = ix.faiss_index.get_state()
    for key in ("centroids", "sq_trained", "list_off", "ids", "codes8"):
        assert np.asarray(after[key]).tobytes() == np.asarray(before[key]).tobytes(), key
    D1, M1 = c2.search(x[:9], 7, index_id)
    assert np.array_equal(D0, D1) and M0 == M1
    c2.close()
