"""Range search (`range_search(x, radius)`, faiss semantics made deterministic; include/dfx.h) from the
list scans up to IndexClient.

CPU: the oracle's range search (tests/oracle_range.py, a cut of its k-NN search) at its strict
boundaries, the socket path Index -> IndexServer -> IndexClient on oracle engines, and this file's
`gpu` tests against the emulated library.  GPU: bit parity of (lims, D, I) with the oracle for every
served kind and list-scan family, consistency with `search`, the refusals and the 2^27 limit.
"""
import os
import platform
import shutil
import subprocess
import sys
import threading

import numpy as np
import pytest

from oracle import oracle as O
from tests import oracle_range as R

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
IP, L2 = O.METRIC_IP, O.METRIC_L2
EMU = bool(os.environ.get("DFX_EMU_LIB"))


def _sz(full, emu):
    return emu if EMU else full


# ------------------------------------------------------------------ the oracle (CPU)
@pytest.mark.parametrize("metric", [L2, IP])
def test_oracle_range_search_strict_boundaries(oracle_lib, metric):
    rs = np.random.RandomState(0)
    xb = rs.randn(40, 8).astype(np.float32)
    xb[10:14] = xb[3]                       # duplicated rows: their distances tie
    ix = R.with_range(O.OracleFlat(8, metric))
    ix.add(xb)
    xq = np.concatenate([xb[3:4] + 0.01 * rs.randn(1, 8).astype(np.float32), rs.randn(3, 8).astype(np.float32)])
    D, I = ix.search(xq, 40)
    toward = np.inf if metric == L2 else -np.inf
    better = (lambda a, b: a < b) if metric == L2 else (lambda a, b: a > b)
    for j in (0, 4, 17):                   # j = 4: the tie of the 5 copies of row 3 on query 0
        r = D[0, j]
        lims, Dr, Ir = ix.range_search(xq[:1], r)
        assert not (Dr == r).any(), "a distance equal to the radius is excluded"
        assert lims[1] == int(better(D[0], r).sum())
        lims2, Dr2, Ir2 = ix.range_search(xq[:1], np.nextafter(r, toward, dtype=np.float32))
        assert lims2[1] == int(better(D[0], r).sum() + (D[0] == r).sum()), "the next float includes the ties"
        np.testing.assert_array_equal(Ir2, I[0, :lims2[1]])        # best first, ties by id
    lims, Dr, Ir = ix.range_search(xq, -toward)                     # nothing passes
    assert lims.tolist() == [0] * 5 and Dr.size == 0 and Ir.size == 0
    lims, Dr, Ir = ix.range_search(xq, toward)                      # every vector
    assert lims.tolist() == [0, 40, 80, 120, 160]
    np.testing.assert_array_equal(Dr.reshape(4, 40), D)
    for q in range(4):
        key = Dr[lims[q]:lims[q + 1]] * (1 if metric == L2 else -1)
        assert (np.diff(key) >= 0).all()
    with pytest.raises(RuntimeError, match="NaN"):
        ix.range_search(xq, float("nan"))


def test_oracle_range_search_covers_every_probed_vector(oracle_lib):
    rs = np.random.RandomState(1)
    from tests.conftest import clustered

    x = clustered(rs, 600, 16, ncl=8)
    ix = R.with_range(O.make_index("ivf_flat", 16, metric=L2, nlist=8))
    ix.train(x)
    ix.add(x)
    ix.nprobe = 3
    lims, D, I = ix.range_search(x[:5], np.inf)
    keys, _ = O.coarse(L2, ix.centroids, x[:5], 3)
    sizes = np.diff(ix.list_off)
    assert np.diff(lims).tolist() == [int(sizes[k].sum()) for k in keys]
    assert ix.search_metric == L2


# ------------------------------------------------------------------ sockets, oracle engines (CPU)
@pytest.fixture(scope="module")
def range_cluster():
    from distributed_faiss_b200.server import IndexServer
    from tests.test_host_logic import free_ports, wait_listening
    import tempfile

    tmp = tempfile.TemporaryDirectory()
    ports = free_ports(3)
    servers = []
    for rank, port in enumerate(ports):
        s = IndexServer(rank, tmp.name, engine_factory=R.oracle_engine_factory)
        threading.Thread(target=s.start_blocking, args=(port,), daemon=True).start()
        servers.append(s)
    wait_listening(ports)
    yield {"ports": ports, "servers": servers}
    for s in servers:
        s.stop()
    tmp.cleanup()


def _expected_merge(servers, index_id, xq, radius):
    """each shard's oracle range search, merged per query best first; equal scores keep the shard
    order and then the shard's own order"""
    per = []
    for s in servers:
        ix = s.indexes[index_id]
        lims, D, I = ix.faiss_index.range_search(xq, radius)
        per.append((lims, D, ix.lookup_meta(I), ix.faiss_index.search_metric))
    assert len({p[3] for p in per}) == 1
    sign = -1.0 if per[0][3] == IP else 1.0
    lims_out, D_out, meta_out = [0], [], []
    for q in range(xq.shape[0]):
        entries = []
        for lims, D, meta, _ in per:
            entries += [(D[j], meta[j]) for j in range(lims[q], lims[q + 1])]
        entries.sort(key=lambda e: sign * float(e[0]))            # stable
        D_out += [e[0] for e in entries]
        meta_out += [e[1] for e in entries]
        lims_out.append(len(D_out))
    return np.array(lims_out), np.array(D_out, dtype=np.float32), meta_out, per[0][3]


CLUSTER_CASES = [
    ("flat", dict(index_builder_type="flat", metric="l2"), IP),        # the flat builder is always IP
    ("ivf_dot", dict(index_builder_type="ivf_simple", metric="dot", centroids=4, nprobe=2), IP),
    ("ivf_l2", dict(index_builder_type="ivf_simple", metric="l2", centroids=4, nprobe=2), L2),
    ("knnlm_dot", dict(index_builder_type="knnlm", metric="dot", centroids=4, code_size=8), L2),  # searches in L2
    ("sq8", dict(faiss_factory="IVF{centroids},SQ8", metric="l2", centroids=4, nprobe=3), L2),
]


@pytest.mark.parametrize("name,kw,smetric", CLUSTER_CASES, ids=[c[0] for c in CLUSTER_CASES])
def test_client_range_search_merges_the_shards(oracle_lib, range_cluster, name, kw, smetric):
    from distributed_faiss_b200.index_cfg import IndexCfg
    from tests.test_host_logic import make_client, wait_trained

    rs = np.random.RandomState(7)
    d = 16
    client = make_client(range_cluster["ports"])
    index_id = "r_" + name
    client.create_index(index_id, IndexCfg(dim=d, train_num=280, **kw))
    base = rs.randn(5, d).astype(np.float32)
    for b in range(3):                                      # one batch per shard, near-duplicate groups
        x = (base[rs.randint(0, 5, 300)] + 0.05 * rs.randn(300, d)).astype(np.float32)
        x[:4] = x[4]                                         # exact duplicates: tied distances
        client.add_index_data(index_id, x, [(b, i) for i in range(300)], False)
    wait_trained(client, index_id)
    xq = np.concatenate([x[:3], rs.randn(2, d).astype(np.float32)])
    lims0, D0, _, _ = _expected_merge(range_cluster["servers"], index_id, xq, np.inf if smetric == L2 else -np.inf)
    some = np.median(D0)                                     # a radius with some results per query
    for radius in (some, np.inf if smetric == L2 else -np.inf, -np.inf if smetric == L2 else np.inf):
        lims, D, meta = client.range_search(xq, radius, index_id)
        el, eD, emeta, em = _expected_merge(range_cluster["servers"], index_id, xq, radius)
        assert em == smetric
        np.testing.assert_array_equal(lims, el)
        np.testing.assert_array_equal(D.view(np.int32), eD.view(np.int32))
        assert meta == emeta
    assert 0 < lims0[-1] and all(isinstance(m, tuple) and len(m) == 2 for m in meta[:3])
    client.drop_index(index_id)
    client.close()


@pytest.mark.parametrize("factory,what", [("IVF4,PQ8x4fs", "IVF_PQ_FS"), ("IVF4,PQ4+4", "IVF_PQR"),
                                          ("IVF4,SQ8,RFlat", "flat refinement")])
def test_client_range_search_refusals(oracle_lib, range_cluster, factory, what):
    from distributed_faiss_b200.index_cfg import IndexCfg
    from distributed_faiss_b200.rpc import ServerException
    from tests.test_host_logic import make_client, wait_trained

    rs = np.random.RandomState(3)
    client = make_client(range_cluster["ports"])
    index_id = "r_refused"
    client.create_index(index_id, IndexCfg(faiss_factory=factory, dim=16, metric="l2", train_num=280))
    for _ in range(3):
        client.add_index_data(index_id, rs.randn(300, 16).astype(np.float32), list(range(300)), False)
    wait_trained(client, index_id)
    with pytest.raises(ServerException, match=what):
        client.range_search(rs.randn(2, 16).astype(np.float32), 1.0, index_id)
    client.drop_index(index_id)
    client.close()


# ------------------------------------------------------------------ emulated library (CPU)
EMU_SUBSET = [
    "test_range_parity_matches_oracle[flat-l2]",
    "test_range_parity_matches_oracle[ivf_flat-ip]",
    "test_range_parity_matches_oracle[ivf_pq-m16]",
    "test_range_parity_matches_oracle[ivf_pq-m32-il]",
    "test_range_parity_matches_oracle[ivf_pq4-m16]",
    "test_range_parity_matches_oracle[ivf_sq8]",
    "test_flat_range_one_hit_per_query_across_tiles[0]",
    "test_flat_range_one_hit_per_query_across_tiles[1]",
    "test_range_search_refusals",
    "test_search_after_range_search_is_unchanged",
]


def test_range_search_on_the_emulated_library():
    if shutil.which("g++") is None or platform.machine() != "x86_64":
        pytest.skip("the emulator needs g++ on x86-64")
    sys.path.insert(0, os.path.join(ROOT, "tests", "emu"))
    try:
        import build_emu_lib
    finally:
        sys.path.pop(0)
    env = dict(os.environ, DFX_EMU_LIB=build_emu_lib.build())
    ids = [f"tests/test_range_search.py::{t}" for t in EMU_SUBSET]
    run = subprocess.run([sys.executable, "-m", "pytest", "-m", "gpu", "-q", "-x", "-p", "no:cacheprovider"] + ids,
                         cwd=ROOT, env=env, capture_output=True, text=True, timeout=1500)
    tail = (run.stdout + run.stderr)[-3000:]
    assert run.returncode == 0, tail
    assert f"{len(EMU_SUBSET)} passed" in run.stdout, tail


# ------------------------------------------------------------------ GPU
def _E():
    from distributed_faiss_b200 import engine

    return engine


def _pair(kind, metric, d, n, rs, nlist=8, M=0, nbits=8, nprobe=3, **params):
    """(GpuIndex, oracle with range search, queries): the oracle builds the shard, the GPU imports it"""
    from tests.conftest import clustered
    from tests.oracle_pq_fs import make_index

    E = _E()
    x = clustered(rs, n, d, ncl=max(nlist, 4))
    x[1:6] = x[0]                                            # exact duplicates: tied distances
    if kind == "flat":
        o = O.OracleFlat(d, metric)
        o.add(x)
    else:
        o = make_index(kind, d, metric=metric, nlist=nlist, M=M, nbits=nbits)
        o.train_niter = 2
        o.train(x[:min(n, 2000)])
        o.add(x)
        o.nprobe = nprobe
    o = R.with_range(o)
    kinds = {"flat": E.KIND_FLAT, "ivf_flat": E.KIND_IVF_FLAT, "ivf_pq": E.KIND_IVF_PQ, "ivf_sq": E.KIND_IVF_SQ16,
             "ivf_sq8": E.KIND_IVF_SQ8}
    g = E.GpuIndex(kinds[kind], d, metric, nlist=nlist if kind != "flat" else 0, pq_m=M, pq_nbits=nbits)
    for k_, v in params.items():
        g.set_param(k_, v)
    g.set_state(o.get_state())
    if kind != "flat":
        g.nprobe = nprobe
    xq = np.concatenate([x[:2], x[0:1] + 0.01, clustered(rs, 4, d, ncl=4)]).astype(np.float32)
    return g, o, xq


def _radii(o, xq):
    """no result, a few (segments shorter than the 2048 sorted in shared memory), some, every probed vector"""
    lims, D, _ = o.range_search(xq, np.inf if o.search_metric == L2 else -np.inf)
    few = np.sort(D)[len(D) // 100]
    if o.search_metric == L2:
        return [float(D.min()), float(few), float(np.median(D)), np.inf]
    return [float(D.max()), float(-np.sort(-D)[len(D) // 100]), float(np.median(D)), -np.inf]


def _assert_same(got, want, what):
    (gl, gD, gI), (wl, wD, wI) = got, want
    np.testing.assert_array_equal(gl, wl, err_msg=what + ": lims")
    np.testing.assert_array_equal(gI, wI, err_msg=what + ": I")
    np.testing.assert_array_equal(gD.view(np.int32), wD.view(np.int32), err_msg=what + ": D bits")


PARITY = {
    "flat-ip": dict(kind="flat", metric=IP, d=8, n=_sz(33000, 32800)),   # two 32768-column tiles
    "flat-l2": dict(kind="flat", metric=L2, d=8, n=_sz(33000, 32800)),
    "ivf_flat-ip": dict(kind="ivf_flat", metric=IP, d=16, n=600),
    "ivf_flat-l2": dict(kind="ivf_flat", metric=L2, d=16, n=600),
    "ivf_pq-m16": dict(kind="ivf_pq", metric=L2, d=32, n=600, M=16),
    "ivf_pq-m32-il": dict(kind="ivf_pq", metric=L2, d=64, n=600, M=32, interleaved=1),
    "ivf_pq-m32-rm": dict(kind="ivf_pq", metric=L2, d=64, n=600, M=32, interleaved=0),
    "ivf_pq-m96": dict(kind="ivf_pq", metric=L2, d=96, n=600, M=96),
    "ivf_pq-m128": dict(kind="ivf_pq", metric=IP, d=128, n=600, M=128),   # IP coarse quantizer, L2 search
    "ivf_pq4-m16": dict(kind="ivf_pq", metric=L2, d=32, n=600, M=16, nbits=4),
    "ivf_sq": dict(kind="ivf_sq", metric=L2, d=16, n=600),
    "ivf_sq8": dict(kind="ivf_sq8", metric=IP, d=16, n=600),
}


@pytest.mark.gpu
@pytest.mark.parametrize("case", list(PARITY))
def test_range_parity_matches_oracle(oracle_lib, case):
    rs = np.random.RandomState(11)
    g, o, xq = _pair(rs=rs, **PARITY[case])
    assert g.search_metric == o.search_metric
    for r in _radii(o, xq):
        _assert_same(g.range_search(xq, r), o.range_search(xq, r), f"{case} radius={r}")
    lims, _, _ = g.range_search(xq, _radii(o, xq)[0])
    assert lims[-1] == 0
    if case.startswith("ivf"):
        st = g.last_stats()
        assert st["nq"] == xq.shape[0] and st["ndis"] == o.range_search(xq, np.inf if o.search_metric == L2 else
                                                                        -np.inf)[0][-1]


@pytest.mark.gpu
def test_range_parity_across_query_chunks(oracle_lib):
    """a flat batch of 1025 queries spans two query chunks (1024 queries each)"""
    rs = np.random.RandomState(12)
    g, o, _ = _pair("flat", L2, 4, 300, rs)
    xq = rs.randn(1025, 4).astype(np.float32)
    for r in (0.5, np.inf):
        _assert_same(g.range_search(xq, r), o.range_search(xq, r), f"flat chunks radius={r}")


@pytest.mark.gpu
@pytest.mark.parametrize("metric", [L2, IP])
def test_flat_range_one_hit_per_query_across_tiles(oracle_lib, metric):
    """database rows as queries at a tight radius, one hit each (the near-duplicate lookup): the hits of
    the first and third query are in the second 32768-column tile, those of the others in the first, so
    the tiles' pieces interleave the queries although no query has more than one result"""
    E = _E()
    rs = np.random.RandomState(18)
    n, d = _sz(33000, 32800), 8
    xb = rs.randn(n, d).astype(np.float32)
    xb /= np.linalg.norm(xb, axis=1, keepdims=True)          # unit rows: only the row itself is that close
    o = R.with_range(O.OracleFlat(d, metric))
    o.add(xb)
    g = E.GpuIndex(E.KIND_FLAT, d, metric)
    g.set_state(o.get_state())
    rows = [n - 10, 5, n - 3, 7]
    radius = 1e-3 if metric == L2 else 0.999
    got = g.range_search(xb[rows], radius)
    _assert_same(got, o.range_search(xb[rows], radius), f"one hit per query, metric {metric}")
    assert got[0].tolist() == [0, 1, 2, 3, 4] and got[2].tolist() == rows


@pytest.mark.gpu
def test_ivf_range_parity_across_query_chunks(oracle_lib):
    """nlist = 32768 on the FFMA coarse quantizer: 1024 queries per chunk, so 1100 queries take two"""
    if EMU:
        pytest.skip("a 32768-list coarse quantizer over 1100 queries is too large for the emulator")
    rs = np.random.RandomState(13)
    d, nlist = 8, 32768
    cent = rs.randn(nlist, d).astype(np.float32)
    x = (cent[rs.randint(0, nlist, 60000)] + 0.05 * rs.randn(60000, d)).astype(np.float32)
    o = R.with_range(O.make_index("ivf_flat", d, metric=L2, nlist=nlist))
    o.centroids = cent
    o.is_trained = True
    o.add(x)
    o.nprobe = 4
    E = _E()
    g = E.GpuIndex(E.KIND_IVF_FLAT, d, L2, nlist=nlist)
    g.set_param("tensor_cores", 0)
    g.set_state(o.get_state())
    g.nprobe = 4
    xq = (x[:1100] + 0.01 * rs.randn(1100, d)).astype(np.float32)
    for r in (0.02, np.inf):
        _assert_same(g.range_search(xq, r), o.range_search(xq, r), f"ivf chunks radius={r}")


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["flat-l2", "ivf_flat-ip", "ivf_pq-m16", "ivf_sq8"])
def test_range_search_equals_cut_search(case):
    """range_search(r) == search(k = 4096) cut at r where no query probes more than 4096 vectors"""
    rs = np.random.RandomState(14)
    spec = dict(PARITY[case], n=3000)
    g, o, xq = _pair(rs=rs, **spec)
    D, I = g.search(xq, 4096)
    assert (I[:, -1] < 0).all(), "every query probes fewer than 4096 vectors"
    ip = g.search_metric == IP
    for r in _radii(o, xq):
        keep = (I >= 0) & ((D > np.float32(r)) if ip else (D < np.float32(r)))
        lims, Dr, Ir = g.range_search(xq, r)
        np.testing.assert_array_equal(np.diff(lims), keep.sum(axis=1))
        np.testing.assert_array_equal(Ir, I[keep])
        np.testing.assert_array_equal(Dr.view(np.int32), D[keep].view(np.int32))


@pytest.mark.gpu
def test_range_search_refusals():
    E = _E()
    rs = np.random.RandomState(15)
    x = rs.randn(512, 16).astype(np.float32)
    cases = [(dict(kind=E.KIND_IVF_PQ_FS, pq_m=8, pq_nbits=4), "IVF_PQ_FS"),
             (dict(kind=E.KIND_IVF_PQR, pq_m=8, refine_m=8), "IVF_PQR"),
             (dict(kind=E.KIND_IVF_SQ8, refine_flat=True), "flat refinement")]
    for kw, what in cases:
        g = E.GpuIndex(d=16, metric=L2, nlist=4, **kw)
        g.set_param("kmeans_niter", 2)
        g.train(x)
        g.add(x)
        n0 = E.launch_count()
        with pytest.raises(RuntimeError, match=what):
            g.range_search(x[:3], 1.0)
        assert E.launch_count() == n0, f"{what}: refused after launching"
    g = E.GpuIndex(E.KIND_IVF_FLAT, 16, L2, nlist=4)
    with pytest.raises(RuntimeError, match="index is not trained"):
        g.range_search(x[:3], 1.0)
    g.set_param("kmeans_niter", 2)
    g.train(x)
    g.add(x)
    with pytest.raises(RuntimeError, match="NaN"):
        g.range_search(x[:3], float("nan"))
    lims, D, I = g.range_search(x[:3], np.inf)
    assert lims[0] == 0 and lims[-1] == I.size > 0
    lims, D, I = g.range_search(x[:0], np.inf)
    assert lims.tolist() == [0] and D.size == 0


@pytest.mark.gpu
def test_range_search_result_limit():
    """2^27 results per call: 1025 queries x 131072 rows raises once counted; the shard stays usable"""
    if EMU:
        pytest.skip("134 million results are too many for the emulator")
    E = _E()
    rs = np.random.RandomState(16)
    xb = rs.randn(131072, 4).astype(np.float32)
    g = E.GpuIndex(E.KIND_FLAT, 4, L2)
    g.add(xb)
    xq = rs.randn(1025, 4).astype(np.float32)
    D0, I0 = g.search(xq[:8], 10)
    with pytest.raises(RuntimeError, match="134217728"):
        g.range_search(xq, np.inf)
    D1, I1 = g.search(xq[:8], 10)
    np.testing.assert_array_equal(I0, I1)
    np.testing.assert_array_equal(D0, D1)
    lims, D, I = g.range_search(xq[:2], np.inf)
    assert lims.tolist() == [0, 131072, 262144]


@pytest.mark.gpu
def test_search_after_range_search_is_unchanged(oracle_lib):
    rs = np.random.RandomState(17)
    for case in ("ivf_pq-m16", "flat-ip"):
        spec = dict(PARITY[case], n=600)
        g, o, xq = _pair(rs=rs, **spec)
        D0, I0 = g.search(xq, 50)
        g.range_search(xq, np.inf if g.search_metric == L2 else -np.inf)
        D1, I1 = g.search(xq, 50)
        np.testing.assert_array_equal(I0, I1)
        np.testing.assert_array_equal(D0.view(np.int32), D1.view(np.int32))
        Do, Io = o.search(xq, 50)
        np.testing.assert_array_equal(I1, Io)
