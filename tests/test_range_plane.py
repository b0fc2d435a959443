"""IndexClient.range_search over the search plane (spmd.SearchPlane, OP_RANGE) and its device merge
(dfx_range_merge_dev), with and without `return_embeddings`.

CPU: a numpy restatement of the device merge (co-ranking) against the socket path's `lexsort` merge of
IndexClient.range_search; the plane at world size 2 on gloo with oracle engines, answer for answer equal to
the sockets; the refusals; the merge kernel on the emulated library.  GPU: `range_search_dev` against
`range_search`, `range_merge_dev` against the restatement, and 4 servers on cuda:0, plane == sockets bit for
bit over every served kind, with the refusals and the per-call bound.  The multi-GPU NCCL form of the
exchange is the gloo test's protocol; it needs more than one GPU to run."""
import os
import platform
import shutil
import subprocess
import sys
import tempfile
import threading

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMU = bool(os.environ.get("DFX_EMU_LIB"))
IP, L2 = 0, 1


# ------------------------------------------------------------------ the merge, restated (CPU)
def restate_merge(lims, D, P, maximize):
    """The device merge restated: each entry's slot is its query's merged offset, plus its rank in its own
    run, plus per other shard the entries of that shard's run for the query that come first (not worse
    when the shard is earlier, strictly better when later).  lims int64[S, nq + 1]; D, P shard-major."""
    S, nq1 = lims.shape
    nq = nq1 - 1
    base = np.concatenate([[0], np.cumsum(lims[:, nq])])
    out_lims = np.zeros(nq + 1, dtype=np.int64)
    np.cumsum((lims[:, 1:] - lims[:, :-1]).sum(axis=0), out=out_lims[1:])
    T = int(base[-1])
    outD = np.empty(T, dtype=np.float32)
    outP = np.empty(T, dtype=np.int64)
    order = np.empty(T, dtype=np.int64)
    key = -D if maximize else D            # ascending in key; -0 == +0 as floats
    for q in range(nq):
        slot0 = out_lims[q]
        runs = [key[base[s] + lims[s, q]:base[s] + lims[s, q + 1]] for s in range(S)]
        for s in range(S):
            idx = base[s] + lims[s, q] + np.arange(runs[s].size)
            slot = slot0 + np.arange(runs[s].size)
            for s2 in range(S):
                if s2 != s:
                    slot = slot + np.searchsorted(runs[s2], runs[s], side="right" if s2 < s else "left")
            outD[slot], outP[slot], order[slot] = D[idx], P[idx], idx
    return out_lims, outD, outP, order


def random_runs(rs, S, nq, maximize, max_len=6, values=(-1.0, -0.0, 0.0, 0.5, 1.0, 2.0)):
    """S shards' sorted runs (best first) of quantized scores: heavy cross-shard ties and +-0"""
    lims = np.zeros((S, nq + 1), dtype=np.int64)
    Ds = []
    for s in range(S):
        for q in range(nq):
            n = int(rs.randint(0, max_len + 1)) if rs.rand() > 0.2 else 0
            v = np.asarray(values, dtype=np.float32)[rs.randint(0, len(values), n)]
            v = v[np.argsort(-v if maximize else v, kind="stable")]
            Ds.append(v)
            lims[s, q + 1] = lims[s, q] + n
    D = np.concatenate(Ds).astype(np.float32) if Ds else np.zeros(0, np.float32)
    return lims, D


class _FakeShard:
    def __init__(self, lims, D, meta, metric, embs=None):
        self.r = (lims, D, meta, metric) + ((embs,) if embs is not None else ())

    def range_search(self, index_id, query, radius, return_embeddings=False):
        return self.r


def _socket_merge(lims, D, maximize, d=3):
    """IndexClient.range_search's own merge (the socket path) over shards answering these runs"""
    from distributed_faiss_b200.client import IndexClient

    S, nq1 = lims.shape
    base = np.concatenate([[0], np.cumsum(lims[:, -1])])
    rows = np.arange(base[-1] * d, dtype=np.float32).reshape(-1, d)
    shards = [_FakeShard(lims[s], D[base[s]:base[s + 1]], list(range(base[s], base[s + 1])), IP if maximize else L2,
                         rows[base[s]:base[s + 1]]) for s in range(S)]
    c = object.__new__(IndexClient)
    c.plane = None
    c._all = lambda fn: [fn(s) for s in shards]
    return c.range_search(np.zeros((nq1 - 1, d), np.float32), 0.0, "x", return_embeddings=True), rows


@pytest.mark.parametrize("maximize", [False, True])
@pytest.mark.parametrize("S,nq", [(1, 5), (2, 9), (5, 7), (3, 0), (4, 1)])
def test_merge_restatement_equals_socket_merge(S, nq, maximize):
    rs = np.random.RandomState(S * 31 + nq + int(maximize))
    for _ in range(5):
        lims, D = random_runs(rs, S, nq, maximize)
        P = np.arange(D.size, dtype=np.int64) * 7 + 3
        ml, mD, mP, order = restate_merge(lims, D, P, maximize)
        (sl, sD, smeta, sE), rows = _socket_merge(lims, D, maximize)
        np.testing.assert_array_equal(ml, sl)
        np.testing.assert_array_equal(mD.view(np.int32), sD.view(np.int32))
        assert order.tolist() == smeta
        np.testing.assert_array_equal(mP, P[order])
        np.testing.assert_array_equal(rows[order], sE)


def test_merge_restatement_edge_cases():
    lims = np.zeros((3, 4), dtype=np.int64)                   # nothing anywhere
    ml, mD, mP, order = restate_merge(lims, np.zeros(0, np.float32), np.zeros(0, np.int64), False)
    assert ml.tolist() == [0, 0, 0, 0] and mD.size == mP.size == order.size == 0
    # -0 and +0 tie: shard order decides, and the bits travel unchanged
    lims = np.array([[0, 1], [0, 1]], dtype=np.int64)
    D = np.array([0.0, -0.0], dtype=np.float32)
    for maximize in (False, True):
        _, mD, _, order = restate_merge(lims, D, np.arange(2, dtype=np.int64), maximize)
        assert order.tolist() == [0, 1] and mD.view(np.int32).tolist() == D.view(np.int32).tolist()


# ------------------------------------------------------------------ gloo world 2, oracle engines (CPU)
def _oracle_range_backend():
    import torch

    from tests.oracle_engine import OracleBackend

    class OracleRangeBackend(OracleBackend):
        """OracleBackend with the plane's range calls: the oracle's range search, the numpy merge"""

        def range_local(self, shard, x_t, radius, embs):
            lims, D, I = shard.range_search(x_t.numpy(), radius)
            R = torch.from_numpy(shard.reconstruct_rows(I).reshape(len(I), x_t.shape[1])) if embs else None
            return torch.from_numpy(lims), torch.from_numpy(D), torch.from_numpy(I), R

        def range_merge(self, lims_t, D_t, P_t, maximize):
            return tuple(torch.from_numpy(a) for a in restate_merge(lims_t.numpy(), D_t.numpy(), P_t.numpy(),
                                                                    maximize))

    return OracleRangeBackend()


def _same(a, b, embs):
    np.testing.assert_array_equal(a[0], b[0])
    np.testing.assert_array_equal(np.asarray(a[1]).view(np.int32), np.asarray(b[1]).view(np.int32))
    assert list(a[2]) == list(b[2])
    if embs:
        np.testing.assert_array_equal(a[3], b[3])


def _worker(rank, world, port, ports, outdir):
    sys.path.insert(0, ROOT)
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world),
                      LOCAL_RANK=str(rank))
    import time

    import torch
    import torch.distributed as dist

    from distributed_faiss_b200 import client as client_mod
    from distributed_faiss_b200 import rpc, spmd
    from distributed_faiss_b200.client import IndexClient
    from distributed_faiss_b200.index_cfg import IndexCfg
    from distributed_faiss_b200.index_state import IndexState
    from distributed_faiss_b200.server import IndexServer
    from tests import oracle_range as R
    from tests.oracle_engine import oracle_merge

    client_mod.ResultHeap.merge_backend = staticmethod(oracle_merge)
    spmd.init_process_group_from_env(backend="gloo")
    s_loc = len(ports) // world
    servers = []
    for j in range(s_loc):
        sr = rank * s_loc + j
        srv = IndexServer(sr, os.path.join(outdir, "store"), engine_factory=R.oracle_engine_factory)
        threading.Thread(target=srv.start_blocking, args=(ports[sr],), daemon=True).start()
        servers.append(srv)
    plane = spmd.SearchPlane(servers, backend=_oracle_range_backend(), device=torch.device("cpu"))
    dist.barrier()
    if rank != 0:
        plane.serve_forever()
        dist.barrier()
        dist.destroy_process_group()
        return

    from tests.test_plane import _wait_listening

    _wait_listening(ports)
    disc = os.path.join(outdir, "servers.txt")
    with open(disc, "w") as fh:
        fh.write(f"{len(ports)}\n" + "".join(f"127.0.0.1,{p}\n" for p in ports))
    client = IndexClient(disc)
    assert client.plane is plane
    rs = np.random.RandomState(5)
    d = 16

    def wait_trained(index_id):
        t0 = time.time()
        while client.get_state(index_id) != IndexState.TRAINED:
            assert time.time() - t0 < 60
            time.sleep(0.02)

    def both_ways(fn):
        client.plane = plane
        try:
            a = fn()
        finally:
            client.detach_plane()
        b = fn()
        client.plane = plane
        return a, b

    def odd_block_radius(name, xq, dists):
        """a radius at which the rank with the most hits has an odd count: with an odd d its block of rows
        ends 4 bytes past an 8-byte boundary"""
        for r in np.quantile(dists, np.linspace(0.05, 0.95, 19)):
            per_server = [int(sub.range_search(name, xq, float(r))[0][-1]) for sub in client.sub_indexes]
            per_rank = [sum(per_server[k * 2:k * 2 + 2]) for k in range(world)]
            if max(per_rank) % 2 == 1:
                return float(r)
        raise AssertionError("no radius with an odd largest block")

    cases = [("ip_odd_d", dict(index_builder_type="flat", metric="dot"), "int", IP, 5),
             ("l2_int", dict(index_builder_type="ivf_simple", metric="l2", centroids=4, nprobe=3), "int", L2, d),
             ("ip_obj", dict(index_builder_type="flat", metric="dot"), "obj", IP, d)]   # last: xq is used below
    for name, kw, meta_kind, smetric, dc in cases:
        base = rs.randn(6, dc).astype(np.float32)
        client.create_index(name, IndexCfg(dim=dc, train_num=200, **kw))
        nxt = 0
        for b in range(8):
            x = (base[rs.randint(0, 6, 60)] + 0.1 * rs.randn(60, dc)).astype(np.float32)
            x[:3] = x[3]                                              # exact duplicates: tied scores
            meta = list(range(nxt, nxt + 60)) if meta_kind == "int" else [(b, i, "m") for i in range(60)]
            client.add_index_data(name, x, meta, False)
            nxt += 60
        client.sync_train(name)
        wait_trained(name)
        xq = np.concatenate([x[:3], base[:2], np.full((1, dc), 50.0, np.float32)])   # the last: no hit anywhere
        full, _ = both_ways(lambda: client.range_search(xq, np.inf if smetric == L2 else -np.inf, name))
        mid = float(np.median(full[1]))
        radii = (mid, np.inf, -np.inf) + ((odd_block_radius(name, xq, full[1]),) if dc % 2 else ())
        for radius in radii:
            for embs in (False, True):
                a, b = both_ways(lambda: client.range_search(xq, radius, name, return_embeddings=embs))
                assert len(a) == len(b) == (4 if embs else 3)
                _same(a, b, embs)
                if embs:
                    assert a[3].shape == (a[0][-1], dc) and a[3].dtype == np.float32
        a, _ = both_ways(lambda: client.range_search(xq, mid, name))
        assert a[0][-2] > 0, "some hits"
        if smetric == L2:
            assert a[0][-1] == a[0][-2], "the far query has no hit"
        if meta_kind == "obj":
            assert all(isinstance(m, tuple) for m in a[2])

    # refusals: the socket path's messages, no hang, and the plane answers afterwards
    client.create_index("fs", IndexCfg(faiss_factory="IVF4,PQ8x4fs", dim=d, metric="l2", train_num=200))
    for _ in range(4):
        client.add_index_data("fs", rs.randn(80, d).astype(np.float32), list(range(80)), False)
    client.sync_train("fs")
    wait_trained("fs")
    for use_plane in (True, False):
        client.plane = plane if use_plane else None
        with pytest.raises(rpc.ServerException, match="IVF_PQ_FS"):
            client.range_search(xq, 1.0, "fs")
    client.plane = plane
    # a mixed-metric index: server 0 flat (inner product), the others IVF-Flat under L2
    for i, sub in enumerate(client.sub_indexes):
        cfg = IndexCfg(dim=d, train_num=50, **(dict(index_builder_type="flat", metric="dot") if i == 0 else
                                               dict(index_builder_type="ivf_simple", metric="l2", centroids=2,
                                                    nprobe=2)))
        sub.create_index("mixed", cfg)
        sub.add_index_data("mixed", rs.randn(60, d).astype(np.float32), list(range(60)), False)
        sub.sync_train("mixed")
    wait_trained("mixed")
    msgs = []
    for use_plane in (True, False):
        client.plane = plane if use_plane else None
        with pytest.raises(RuntimeError, match="different search metrics") as ei:
            client.range_search(xq, 1.0, "mixed")
        assert not isinstance(ei.value, rpc.ServerException)
        msgs.append(str(ei.value))
    assert msgs[0] == msgs[1]
    client.plane = plane
    client.cfg = IndexCfg(metric="dot")
    D, M = client.search(xq, 5, "ip_obj")
    assert D.shape == (6, 5)
    lims, _, _ = client.range_search(xq, -np.inf, "ip_obj")
    assert lims[-1] == 6 * 480
    np.savez(os.path.join(outdir, "done.npz"), ok=np.array([1]))
    client.close()
    plane.stop()
    dist.barrier()
    dist.destroy_process_group()


def test_range_search_over_gloo_plane_equals_sockets():
    import torch.multiprocessing as mp

    from tests.test_plane import _free_ports

    world = 2
    ports = _free_ports(5)
    with tempfile.TemporaryDirectory() as outdir:
        mp.spawn(_worker, args=(world, ports[0], ports[1:], outdir), nprocs=world, join=True)
        assert os.path.exists(os.path.join(outdir, "done.npz"))


# ------------------------------------------------------------------ emulated library (CPU)
EMU_SUBSET = [
    "test_range_merge_dev_matches_restatement[1]",
    "test_range_merge_dev_matches_restatement[2]",
    "test_range_merge_dev_matches_restatement[7]",
]


def test_range_merge_on_the_emulated_library():
    if shutil.which("g++") is None or platform.machine() != "x86_64":
        pytest.skip("the emulator needs g++ on x86-64")
    sys.path.insert(0, os.path.join(ROOT, "tests", "emu"))
    try:
        import build_emu_lib
    finally:
        sys.path.pop(0)
    env = dict(os.environ, DFX_EMU_LIB=build_emu_lib.build())
    ids = [f"tests/test_range_plane.py::{t}" for t in EMU_SUBSET]
    run = subprocess.run([sys.executable, "-m", "pytest", "-m", "gpu", "-q", "-x", "-p", "no:cacheprovider"] + ids,
                         cwd=ROOT, env=env, capture_output=True, text=True, timeout=1500)
    tail = (run.stdout + run.stderr)[-3000:]
    assert run.returncode == 0, tail
    assert f"{len(EMU_SUBSET)} passed" in run.stdout, tail


# ------------------------------------------------------------------ GPU
def _device_merge(lims, D, P, maximize):
    """dfx_range_merge_dev on CUDA tensors; on the emulated library (no CUDA tensors) on host buffers,
    which are its device memory"""
    from distributed_faiss_b200 import engine as E

    if not EMU:
        import torch

        out = E.range_merge_dev(torch.from_numpy(lims).cuda(), torch.from_numpy(D).cuda(), torch.from_numpy(P).cuda(),
                                maximize)
        return tuple(t.cpu().numpy() for t in out)
    import ctypes as C

    S, nq1 = lims.shape
    T = D.size
    lims, D, P = (np.ascontiguousarray(a) for a in (lims, D, P))
    ol, oD, oP, order = (np.empty(nq1, np.int64), np.empty(T, np.float32), np.empty(T, np.int64),
                         np.empty(T, np.int64))
    ptr = E._np_ptr
    E._check(E.lib().dfx_range_merge_dev(C.c_int64(S), C.c_int64(nq1 - 1), ptr(lims), ptr(D), ptr(P), C.c_int64(T),
                                         C.c_int(1 if maximize else 0), ptr(ol), ptr(oD), ptr(oP), ptr(order), None))
    return ol, oD, oP, order


@pytest.mark.gpu
@pytest.mark.parametrize("S", [1, 2, 7])
def test_range_merge_dev_matches_restatement(S):
    rs = np.random.RandomState(40 + S)
    long_len = 300 if EMU else 5200
    for maximize in (False, True):
        for nq, max_len in ((1, long_len), (37, 12), (300, 40), (4, 0)):
            lims, D = random_runs(rs, S, nq, maximize, max_len=max_len,
                                  values=np.round(rs.randn(16), 1).tolist() + [0.0, -0.0])
            P = rs.randint(-5, 1 << 40, D.size, dtype=np.int64)
            got = _device_merge(lims, D, P, maximize)
            want = restate_merge(lims, D, P, maximize)
            np.testing.assert_array_equal(got[0], want[0])
            np.testing.assert_array_equal(got[1].view(np.int32), want[1].view(np.int32))
            np.testing.assert_array_equal(got[2], want[2])
            np.testing.assert_array_equal(got[3], want[3])


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["flat-l2", "ivf_flat-ip", "ivf_pq-m16", "ivf_sq8"])
def test_range_search_dev_equals_range_search(oracle_lib, case):
    import torch

    from tests.test_range_search import PARITY, _pair, _radii

    rs = np.random.RandomState(21)
    g, o, xq = _pair(rs=rs, **dict(PARITY[case], n=3000))
    for r in _radii(o, xq):
        want = g.range_search(xq, r)
        got = [t.cpu().numpy() for t in g.range_search_dev(torch.from_numpy(xq).cuda(), r)]
        np.testing.assert_array_equal(got[0], want[0])
        np.testing.assert_array_equal(got[2], want[2])
        np.testing.assert_array_equal(got[1].view(np.int32), want[1].view(np.int32))


PLANE_KINDS = [
    ("flat_ip", dict(index_builder_type="flat", metric="dot"), 64),
    ("flat_l2", dict(faiss_factory="Flat", metric="l2"), 64),
    ("ivf_flat_ip", dict(index_builder_type="ivf_simple", metric="dot", centroids=16, nprobe=4), 64),
    ("ivf_pq32", dict(index_builder_type="knnlm", metric="l2", centroids=16, code_size=32), 128),
    ("ivf_pq4", dict(index_builder_type="knnlm", metric="l2", centroids=16, code_size=16, bits_per_vector=4), 64),
    ("ivf_sq8", dict(faiss_factory="IVF16,SQ8", metric="l2", centroids=16, nprobe=4), 64),
    ("sqfp16", dict(faiss_factory="SQfp16", metric="l2"), 64),
    ("pq16", dict(faiss_factory="PQ16", metric="dot"), 64),
]


@pytest.mark.gpu
def test_range_search_plane_equals_sockets_on_gpu():
    """4 servers on cuda:0: the plane and the sockets return the same (lims, scores, meta, embs) bit for bit"""
    from distributed_faiss_b200.index_cfg import IndexCfg
    from tests.test_gpu_api import _both_ways, _plane_cluster, wait_trained

    store, servers, plane, client = _plane_cluster(4)
    rs = np.random.RandomState(23)
    try:
        for name, kw, d in PLANE_KINDS:
            client.create_index(name, IndexCfg(dim=d, train_num=2000, **kw))
            centers = rs.randn(20, d).astype(np.float32)
            nxt = 0
            for b in range(4):
                x = (centers[rs.randint(0, 20, 800)] + 0.3 * rs.randn(800, d)).astype(np.float32)
                x[:4] = x[4]
                meta = list(range(nxt, nxt + 800)) if b != 3 or name != "flat_l2" else [(i,) for i in range(800)]
                client.add_index_data(name, x, meta, False)
                nxt += 800
            client.sync_train(name)
            wait_trained(client, name)
            if "nprobe" not in kw and "centroids" in kw:
                client.set_nprobe(name, 6)
            xq = np.concatenate([x[:3], (centers[:5] + 0.3 * rs.randn(5, d)).astype(np.float32)])
            smetric = servers[0].indexes[name].search_metric()
            worst = np.inf if smetric == L2 else -np.inf
            full, _ = _both_ways(client, plane, lambda: client.range_search(xq, worst, name))
            if "centroids" not in kw:
                assert (np.diff(full[0]) > 2048).all(), "merged segments beyond 2048 hits"
            pct = float(np.percentile(full[1], 5 if smetric == L2 else 95))
            for radius in (pct, worst, -worst):
                for embs in (False, True):
                    a, b = _both_ways(client, plane, lambda: client.range_search(xq, radius, name, embs))
                    _same(a, b, embs)
            a, _ = _both_ways(client, plane, lambda: client.range_search(xq, pct, name))
            assert 0 < a[0][-1] < full[0][-1]
    finally:
        client.close()
        plane.stop()
        for s in servers:
            s.stop()
        store.cleanup()


@pytest.mark.gpu
def test_range_search_plane_refusals_on_gpu():
    import torch

    from distributed_faiss_b200 import engine as E
    from distributed_faiss_b200 import rpc
    from distributed_faiss_b200.index_cfg import IndexCfg
    from tests.test_gpu_api import _plane_cluster, wait_trained

    store, servers, plane, client = _plane_cluster(4)
    rs = np.random.RandomState(29)
    d = 16
    xq = rs.randn(3, d).astype(np.float32)
    try:
        client.create_index("ok", IndexCfg(index_builder_type="flat", dim=d, metric="dot", train_num=100))
        for _ in range(4):
            client.add_index_data("ok", rs.randn(200, d).astype(np.float32), list(range(200)), False)
        client.sync_train("ok")
        wait_trained(client, "ok")
        client.cfg = IndexCfg(metric="dot")
        D0, M0 = client.search(xq, 5, "ok")
        L0 = client.range_search(xq, -np.inf, "ok")

        def still_serves():
            client.cfg = IndexCfg(metric="dot")      # create_index of another index replaced it
            D, M = client.search(xq, 5, "ok")
            assert np.array_equal(D, D0) and M == M0
            _same(client.range_search(xq, -np.inf, "ok"), L0, False)

        for factory, what in (("IVF4,PQ8x4fs", "IVF_PQ_FS"), ("IVF4,PQ4+4", "IVF_PQR"),
                              ("IVF4,SQ8,RFlat", "flat refinement")):
            client.create_index(what, IndexCfg(faiss_factory=factory, dim=d, metric="l2", train_num=400))
            for _ in range(4):   # 400 rows per server: IVF-PQR trains its codebooks on at least 256
                client.add_index_data(what, rs.randn(400, d).astype(np.float32), list(range(400)), False)
            client.sync_train(what)
            wait_trained(client, what)
            with pytest.raises(rpc.ServerException, match=what):
                client.range_search(xq, 1.0, what)
            still_serves()
        with pytest.raises(rpc.ServerException, match="NaN"):
            client.range_search(xq, float("nan"), "ok")
        still_serves()
        client.create_index("cold", IndexCfg(index_builder_type="flat", dim=d, train_num=10_000))
        client.add_index_data("cold", rs.randn(10, d).astype(np.float32), list(range(10)), False)
        with pytest.raises(rpc.ServerException, match="not trained"):
            client.range_search(xq, 1.0, "cold")
        still_serves()
        # the per-call bound: two flat shards of 131072 rows, 600 queries: 78.6 M hits each, 157 M together
        n, nq = 131072, 600
        xb = rs.randn(n, 4).astype(np.float32)
        for i, s in enumerate(servers):
            g = E.GpuIndex(E.KIND_FLAT, 4, E.METRIC_L2, device=0)
            g.add(xb if i < 2 else xb[:1])
            s.adopt_index("big", IndexCfg(index_builder_type="flat", dim=4, metric="l2"), g,
                          torch.arange(g.ntotal, dtype=torch.int64, device="cuda:0"))
        with pytest.raises(rpc.ServerException, match="134217728"):
            client.range_search(rs.randn(nq, 4).astype(np.float32), np.inf, "big")
        still_serves()
        lims, _, _ = client.range_search(rs.randn(2, 4).astype(np.float32), np.inf, "big")
        assert lims.tolist() == [0, 2 * n + 2, 4 * n + 4]
        for s in servers:   # adopted shards have no storage directory to be saved into on stop()
            s.indexes.pop("big")
    finally:
        client.close()
        plane.stop()
        for s in servers:
            s.stop()
        store.cleanup()


# ------------------------------------------------------------------ the exchange's layout and decision (CPU)
@pytest.mark.parametrize("d", [1, 3, 5, 16, 768])
@pytest.mark.parametrize("T_max", [0, 1, 7, 1000])
def test_range_exchange_blocks_stay_8_byte_aligned(d, T_max):
    from distributed_faiss_b200 import spmd

    for embs in (False, True):
        off_D, off_P, off_E, stride = spmd.range_layout(3, 11, d, embs, T_max)
        assert off_D % 8 == off_P % 8 == off_E % 8 == stride % 8 == 0
        assert off_P >= off_D + 4 * T_max and off_E >= off_P + 8 * T_max
        assert stride >= off_E + (4 * T_max * d if embs else 0)


def _info(status, free, totals, metrics, msg=b""):
    from distributed_faiss_b200 import spmd

    S_loc = len(totals)
    row = np.zeros(3 + 2 * S_loc + spmd.RANGE_MSG_BYTES // 8, dtype=np.int64)
    row[0], row[1], row[2] = status, len(msg), free
    row[3:3 + S_loc], row[3 + S_loc:3 + 2 * S_loc] = totals, metrics
    row[3 + 2 * S_loc:].view(np.uint8)[:len(msg)] = np.frombuffer(msg, dtype=np.uint8)
    return row


def test_range_decision_refuses_what_does_not_fit():
    from distributed_faiss_b200 import spmd

    big = 1 << 50
    ok = np.stack([_info(0, big, [10, 20], [1, 1]), _info(0, big, [5, 0], [1, 1])])
    assert spmd.range_decide(ok, 2, 4, 8, True) == (spmd.ST_OK, "")
    err = np.stack([_info(0, big, [10, 20], [1, 1]), _info(spmd.ST_ERROR, big, [0, 0], [-1, -1], b"boom")])
    assert spmd.range_decide(err, 2, 4, 8, False) == (spmd.ST_ERROR, "boom")
    mixed = np.stack([_info(0, big, [1, 1], [0, 0]), _info(0, big, [1, 1], [1, 1])])
    assert spmd.range_decide(mixed, 2, 4, 8, False) == (spmd.ST_RANGE_METRICS, [0, 1])
    many = np.stack([_info(0, big, [spmd.RANGE_MAX_HITS, 0], [1, 1]), _info(0, big, [1, 0], [1, 1])])
    st, msg = spmd.range_decide(many, 2, 4, 8, False)
    assert st == spmd.ST_RANGE_LIMIT and "134217728" in msg
    # 10 M hits of 768-dimensional rows: about 30 GiB of rows each for the gather, the merge and the reorder
    totals = [5_000_000, 0]
    need = spmd.range_need_bytes(2, 2, 1000, 768, True, np.array([totals, totals]))
    assert need > 3 * 10_000_000 * 768 * 4
    tight = np.stack([_info(0, big, totals, [1, 1]), _info(0, need, totals, [1, 1])])
    st, msg = spmd.range_decide(tight, 2, 1000, 768, True)
    assert st == spmd.ST_RANGE_LIMIT and "plane rank 1" in msg and "embeddings" in msg
    assert spmd.range_decide(tight, 2, 1000, 768, False) == (spmd.ST_OK, ""), "without rows it fits"
