"""GPU parity tests: the CUDA path (through the C-ABI, libdfx.so) against the CPU oracle.

Bar (BASELINE.json north_star): returned ids bit-exact at full nprobe, distances within 1e-4.
Because the kernels follow the oracle's canonical summation orders the distances are in fact
required to be BIT-EXACT here (np.array_equal on float32); the 1e-4 tolerance is only used
against the independent float64 restatement (oracle/ref_numpy.py).
"""
import numpy as np
import pytest

from tests.conftest import clustered

pytestmark = pytest.mark.gpu

IP, L2 = 0, 1
# DFX_EMU_LIB: the same tests against the library built for the CPU emulator (tests/emu/); the two
# layout tests shrink their shard there (a fiber-emulated k-means over 30 k vectors takes minutes)
EMU = bool(__import__("os").environ.get("DFX_EMU_LIB"))


def _sz(full, emu):
    return emu if EMU else full


def _engine():
    from distributed_faiss_b200 import engine

    return engine


def _mk_pair(kind, d, metric, nlist=0, M=0):
    """(gpu index, oracle index) of the same configuration"""
    from oracle import oracle as O

    E = _engine()
    kinds = {"flat": E.KIND_FLAT, "ivf_flat": E.KIND_IVF_FLAT, "ivf_pq": E.KIND_IVF_PQ, "ivf_sq": E.KIND_IVF_SQ16}
    g = E.GpuIndex(kinds[kind], d, metric, nlist=nlist, pq_m=M)
    o = O.make_index(kind, d, metric=metric, nlist=nlist, M=M)
    return g, o


def _assert_same(Dg, Ig, Do, Io, what):
    same_i = np.array_equal(Ig, Io)
    same_d = np.array_equal(Dg, Do)
    if not (same_i and same_d):
        bad = np.argwhere((Ig != Io) | (Dg != Do))
        q, j = bad[0]
        raise AssertionError(
            f"{what}: {len(bad)} mismatching slots of {Ig.size}; first at q={q} j={j}: "
            f"gpu=({Dg[q, j]!r},{Ig[q, j]}) oracle=({Do[q, j]!r},{Io[q, j]})\n"
            f"gpu row   D={Dg[q]} I={Ig[q]}\noracle row D={Do[q]} I={Io[q]}")


# ------------------------------------------------------------------ flat
@pytest.mark.parametrize("metric", [IP, L2])
@pytest.mark.parametrize("nq", [1, 7, 33])
def test_flat_matches_oracle(metric, nq):
    rs = np.random.RandomState(1)
    d, n, k = 128, 5000, 10
    xb = rs.rand(n, d).astype(np.float32)
    xq = rs.rand(nq, d).astype(np.float32)
    g, o = _mk_pair("flat", d, metric)
    g.add(xb[:3000]); g.add(xb[3000:])
    o.add(xb)
    assert g.ntotal == n
    _assert_same(*g.search(xq, k), *o.search(xq, k), f"flat metric={metric}")


def test_flat_config1_100k():
    """BASELINE configs[0]: flat d=128, 100k vectors, 1k queries (oracle on a query sample)."""
    rs = np.random.RandomState(0)
    d, n, nq, k = 128, 100_000, 1000, 10
    xb = rs.rand(n, d).astype(np.float32)
    xq = rs.rand(nq, d).astype(np.float32)
    g, o = _mk_pair("flat", d, IP)
    g.add(xb); o.add(xb)
    Dg, Ig = g.search(xq, k)
    sel = np.arange(0, nq, 25)
    Do, Io = o.search(xq[sel], k)
    _assert_same(Dg[sel], Ig[sel], Do, Io, "flat 100k")
    # sortedness + self-consistency at full size
    assert (np.diff(Dg, axis=1) <= 0).all()


def test_flat_edge_cases():
    rs = np.random.RandomState(2)
    d = 32
    g, o = _mk_pair("flat", d, IP)
    xq = rs.rand(3, d).astype(np.float32)
    D, I = g.search(xq, 4)  # empty index
    assert (I == -1).all() and (D == -np.finfo(np.float32).max).all()
    xb = rs.rand(3, d).astype(np.float32)
    xb[2] = xb[0]  # exact duplicate -> tie broken by id
    g.add(xb); o.add(xb)
    _assert_same(*g.search(xq, 5), *o.search(xq, 5), "flat k > ntotal with ties")
    with pytest.raises(RuntimeError, match="xb: wrong size"):
        g.set_array("xb", xb.reshape(-1)[:-1])


# ------------------------------------------------------------------ IVF kinds
def _build_both(kind, metric, d, nlist, M, n, rs, via="gpu"):
    """train+add on one side, ship the state to the other, so that both hold the SAME shard"""
    xb = clustered(rs, n, d, ncl=max(8, nlist // 2))
    g, o = _mk_pair(kind, d, metric, nlist=nlist, M=M)
    if via == "gpu":
        if EMU and kind != "flat":
            g.set_param("kmeans_niter", 2)
        g.train(xb[: n // 2])
        g.add(xb[: n // 3]); g.add(xb[n // 3:])
        st = g.get_state()
        o.set_state(st)
        if kind == "ivf_pq":  # K7: per-vector term computed on device == oracle's
            assert np.array_equal(st["tvals"], o.tvals)
    else:
        o.train(xb[: n // 2])
        o.add(xb)
        g.set_state(o.get_state())
        if kind == "ivf_pq":
            assert np.array_equal(g.get_array("tvals"), o.tvals)
    assert g.ntotal == n == o.ntotal
    return g, o, xb


CASES = [
    ("ivf_flat", L2, 64, 16, 0),
    ("ivf_flat", IP, 64, 16, 0),
    ("ivf_pq", L2, 64, 16, 16),
    ("ivf_pq", L2, 128, 32, 32),
    ("ivf_pq", IP, 128, 16, 32),   # knnlm with metric="dot": IP coarse quantizer, L2 PQ (quirk B2)
    ("ivf_pq", L2, 96, 16, 24),    # generic-M code path
    ("ivf_sq", L2, 64, 16, 0),
    ("ivf_sq", L2, 768, 8, 0),
]


@pytest.mark.parametrize("kind,metric,d,nlist,M", CASES)
@pytest.mark.parametrize("via", ["gpu", "oracle"])
def test_ivf_matches_oracle(kind, metric, d, nlist, M, via):
    rs = np.random.RandomState(3)
    n = 6000
    g, o, xb = _build_both(kind, metric, d, nlist, M, n, rs, via=via)
    xq = np.concatenate([clustered(rs, 20, d, ncl=8), xb[:5] + 0.01 * rs.randn(5, d).astype(np.float32)])
    for nprobe in (nlist, 1, 5):  # full nprobe first: the north-star parity condition
        g.nprobe = nprobe; o.nprobe = nprobe
        for k in (10, 1, 100, 300):  # 300 > 128: the full-width CTA merge path
            Dg, Ig = g.search(xq, k)
            Do, Io = o.search(xq, k)
            _assert_same(Dg, Ig, Do, Io, f"{kind} metric={metric} d={d} via={via} nprobe={nprobe} k={k}")
        assert g.last_stats()["ndis"] == o.last_ndis


@pytest.mark.parametrize("kind,metric,d,nlist,M", [c for c in CASES if c[2] <= 128])
def test_ivf_close_to_float64_restatement(kind, metric, d, nlist, M):
    """GPU distances vs the independent float64 restatement: |dg - d64| <= 1e-4 * scale."""
    from oracle import ref_numpy as R

    rs = np.random.RandomState(4)
    g, o, xb = _build_both(kind, metric, d, nlist, M, 4000, rs)
    xq = clustered(rs, 16, d, ncl=8)
    g.nprobe = nlist
    Dg, Ig = g.search(xq, 10)
    D64, I64 = R.ivf_search(g.get_state(), xq, nlist, 10)
    scale = (xq.astype(np.float64) ** 2).sum(1, keepdims=True) + (xb.astype(np.float64) ** 2).sum(1).max()
    assert (np.abs(Dg - D64) <= 1e-4 * scale).all()
    assert (Ig == I64).mean() > 0.98  # ids differ only where float64 distances are within fp32 rounding


def test_ivf_edge_cases():
    """k > hits (-1 / FLT_MAX padding), empty lists, nprobe > nlist, single-vector lists, ties."""
    from oracle import oracle as O

    rs = np.random.RandomState(5)
    d, nlist = 32, 8
    E = _engine()
    for kind, M in (("ivf_flat", 0), ("ivf_pq", 8), ("ivf_sq", 0)):
        o = O.make_index(kind, d, metric=L2, nlist=nlist, M=M)
        xb = clustered(rs, 600, d, ncl=4, sigma=0.05)  # 4 clusters, 8 lists -> some lists tiny/empty
        xb[10:20] = xb[0]  # exact duplicates -> exact ties
        o.train(xb); o.add(xb[:37])  # few vectors: most lists empty
        kinds = {"ivf_flat": E.KIND_IVF_FLAT, "ivf_pq": E.KIND_IVF_PQ, "ivf_sq": E.KIND_IVF_SQ16}
        g = E.GpuIndex(kinds[kind], d, L2, nlist=nlist, pq_m=M)
        g.set_state(o.get_state())
        xq = xb[:9]
        for nprobe in (1, 3, 50):
            g.nprobe = nprobe; o.nprobe = nprobe
            Dg, Ig = g.search(xq, 64)
            Do, Io = o.search(xq, 64)
            _assert_same(Dg, Ig, Do, Io, f"edge {kind} nprobe={nprobe}")
            assert (Ig == -1).any()
            assert (Dg[Ig == -1] == np.finfo(np.float32).max).all()
        _assert_exchange_refusals(g, o.get_state(), {"ivf_flat": "vecs", "ivf_pq": "codes", "ivf_sq": "codes16"}[kind])


def _import_without(g, st, skip):
    """import every array of the state `st` into `g` but `skip`, then finish the import"""
    E = _engine()
    for name in E.StateLayout(g).arrays:
        if name not in (skip, "tvals"):
            g.set_array(name, st[name])
    E._check(E.lib().dfx_import_done(g._h))


def _assert_exchange_refusals(g, st, payload):
    """what the state exchange of an IVF index `g` holding the state `st` (payload array `payload`,
    8-bit codes) refuses"""
    import ctypes as C

    E = _engine()
    small = np.zeros(2, dtype=np.int64)
    with pytest.raises(RuntimeError, match="output buffer too small for 'ids'"):
        E._check(E.lib().dfx_get_array(g._h, b"ids", E._np_ptr(small), C.c_int64(small.nbytes), None))
    with pytest.raises(RuntimeError, match="no array named 'nope' in this index"):
        E._check(E.lib().dfx_get_array(g._h, b"nope", None, C.c_int64(0), None))

    def fresh():
        return E.GpuIndex(g.kind, g.d, g.metric, nlist=g.nlist, pq_m=g.pq_m, pq_nbits=g.pq_nbits)

    g2 = fresh()
    with pytest.raises(RuntimeError, match="no array named 'centroids' in this index"):
        g2.get_array("centroids")  # not trained yet
    for name in ("nope", "tvals", "xb"):
        with pytest.raises(RuntimeError, match=f"cannot import array '{name}'"):
            E._check(E.lib().dfx_set_array(g2._h, name.encode(), E._np_ptr(small), C.c_int64(small.nbytes)))
    for name in E.StateLayout(g).arrays:
        if name != "tvals":
            with pytest.raises(RuntimeError, match=f"{'payload' if name == payload else name}: wrong size"):
                g2.set_array(name, st[name].reshape(-1)[:-1])
    bad = st["list_off"].copy()
    bad[0] = 1
    with pytest.raises(RuntimeError, match=r"list_off\[0\] must be 0"):
        g2.set_array("list_off", bad)
    g2.set_array("list_off", st["list_off"])
    for v in (-1, 1 << 31):
        bad = st["ids"].copy()
        bad[3] = v
        with pytest.raises(RuntimeError, match=r"ids must be in \[0, 2\^31\)"):
            g2.set_array("ids", bad)
    with pytest.raises(RuntimeError, match="import: centroids and list_off are required"):
        _import_without(fresh(), st, "centroids")
    if "codebooks" in st:
        with pytest.raises(RuntimeError, match="import: codebooks are required"):
            _import_without(fresh(), st, "codebooks")


def test_ivfpq_larger_property():
    """A shard too big for the oracle to scan exhaustively in seconds: compare on a query sample,
    and check size-independent properties on the full batch (sortedness, ids valid and unique,
    batch invariance, idempotence)."""
    rs = np.random.RandomState(6)
    d, nlist, M, n = 128, 256, 32, 300_000
    g, o, xb = _build_both("ivf_pq", L2, d, nlist, M, n, rs)
    xq = xb[rs.randint(0, n, 512)] + 0.02 * rs.randn(512, d).astype(np.float32)
    g.nprobe = 16; o.nprobe = 16
    Dg, Ig = g.search(xq, 10)
    assert (np.diff(Dg, axis=1) >= 0).all()
    assert ((Ig >= 0) & (Ig < n)).all()
    assert all(len(set(r)) == len(r) for r in Ig.tolist())
    D2, I2 = g.search(xq, 10)
    assert np.array_equal(Dg, D2) and np.array_equal(Ig, I2)
    D1, I1 = g.search(xq[100:101], 10)  # batch invariance: same answer alone or in a batch
    assert np.array_equal(D1[0], Dg[100]) and np.array_equal(I1[0], Ig[100])
    sel = np.arange(0, 512, 16)
    Do, Io = o.search(xq[sel], 10)
    _assert_same(Dg[sel], Ig[sel], Do, Io, "ivf_pq 300k sample")


# ------------------------------------------------------------------ K6 merge
def test_merge_reference_golden():
    """golden vectors of reference tests/test_integration.py:181-203"""
    import json, os

    E = _engine()
    gold = json.load(open(os.path.join(os.path.dirname(__file__), "golden", "merge_golden.json")))
    D = np.array(gold["shard_D"], dtype=np.float32)  # [S, nq, k]
    meta = gold["shard_meta"]
    S, nq, k = D.shape
    pos = np.arange(S * nq * k, dtype=np.int64).reshape(S, nq, k)
    flat_meta = [m for s in meta for row in s for m in row]
    for negate, key in ((False, "minimize"), (True, "maximize")):
        outD, outP = E.merge(D, pos, negate=negate)
        assert [flat_meta[p] for p in outP[0]] == gold[key]["meta"][0]
        assert np.allclose(outD[0], np.array(gold[key]["D"][0], dtype=np.float32), rtol=0, atol=0)


@pytest.mark.parametrize("S,nq,k", [(2, 1, 4), (8, 64, 10), (4, 300, 100), (8, 4096, 10), (3, 5, 1)])
def test_merge_matches_oracle(S, nq, k):
    from oracle import oracle as O

    E = _engine()
    rs = np.random.RandomState(7)
    D = np.sort(rs.rand(S, nq, k).astype(np.float32), axis=2)
    D[rs.rand(S, nq, k) < 0.05] = np.finfo(np.float32).max  # shards with missing hits
    D[0, :, : k // 2] = D[1 % S, :, : k // 2]  # cross-shard ties: earlier shard must win
    I = rs.randint(0, 1 << 40, size=(S, nq, k)).astype(np.int64)
    I[D == np.finfo(np.float32).max] = -1
    for negate in (False, True):
        Dx = -D if negate else D
        outD, outI = E.merge(Dx, I, negate=negate)
        pos = np.arange(S * nq * k, dtype=np.int64).reshape(S, nq, k)
        refD, refP = O.merge(-Dx if negate else Dx, pos)
        refI = np.where(refP >= 0, I.reshape(-1)[np.maximum(refP, 0)], -1)
        assert np.array_equal(outD, refD)
        assert np.array_equal(outI, refI)


# ------------------------------------------------------------------ reconstruct / accessors
def test_reconstruct_and_centroids():
    rs = np.random.RandomState(8)
    for kind, M in (("ivf_flat", 0), ("ivf_pq", 16), ("ivf_sq", 0)):
        g, o, xb = _build_both(kind, L2, 64, 16, M, 3000, rs)
        ids = np.array([0, 5, 2999, -1, 17], dtype=np.int64)
        R_g = g.reconstruct_rows(ids)
        R_o = o.reconstruct_rows(ids)
        assert np.isnan(R_g[3]).all()
        ok = [0, 1, 2, 4]
        assert np.allclose(R_g[ok], R_o[ok], rtol=0, atol=1e-6)
        assert np.array_equal(g.quantizer.reconstruct_n(0, 16), o.quantizer.reconstruct_n(0, 16))
        D, I, R = g.search_and_reconstruct(xb[:4], 3)
        assert R.shape == (4, 3, 64)


def test_gpu_training_quality():
    """GPU k-means / PQ training is not bit-comparable to the oracle's (different sampling), but
    its quantisation error must be in the same range as the oracle's on the same data."""
    from oracle import oracle as O

    rs = np.random.RandomState(9)
    d, nlist, M, n = 64, 32, 16, 20000
    xb = clustered(rs, n, d, ncl=40, sigma=0.2)
    g, o = _mk_pair("ivf_pq", d, L2, nlist=nlist, M=M)
    g.train(xb); g.add(xb)
    o.train(xb); o.add(xb)

    def recon_err(ix):
        R = ix.reconstruct_rows(np.arange(0, n, 7, dtype=np.int64))
        return float(((R - xb[::7]) ** 2).sum(1).mean())

    eg, eo = recon_err(g), recon_err(o)
    assert eg < 1.25 * eo + 1e-6, (eg, eo)
    lens = np.diff(g.get_array("list_off"))
    assert lens.sum() == n and (lens > 0).sum() >= nlist // 2


def test_device_pointer_path_matches_host_path():
    """train_dev/add_dev/finalize/search_dev on torch's stream (the NCCL data plane uses these)
    must give the same shard and the same answers as the host-buffer entry points, including
    when host- and device-stream calls are interleaved (regression: cross-stream race)."""
    import torch
    from oracle import oracle as O

    E = _engine()
    rs = np.random.RandomState(11)
    d, nlist, M, n = 128, 64, 32, 50_000
    xb = clustered(rs, n, d, ncl=80)
    xq = xb[:40] + 0.01 * rs.randn(40, d).astype(np.float32)
    g = E.GpuIndex(E.KIND_IVF_PQ, d, L2, nlist=nlist, pq_m=M)
    xb_t = torch.from_numpy(xb).cuda()
    g.train_dev(xb_t[:20000].contiguous())
    for i0 in range(0, n, 12500):
        g.add_dev(xb_t[i0:i0 + 12500].contiguous())
    g.finalize()  # host-side call right behind asynchronous device-stream work
    assert g.ntotal == n
    o = O.OracleIVFPQ(d, nlist, M, 8, coarse_metric=L2)
    o.set_state(g.get_state())
    # the shard built through the device path holds what the oracle would have built from the
    # same trained state: same assignment, same codes
    o2 = O.OracleIVFPQ(d, nlist, M, 8, coarse_metric=L2)
    o2.centroids, o2.codebooks, o2.is_trained = o.centroids, o.codebooks, True
    o2.add(xb)
    assert np.array_equal(o2.list_off, o.list_off)
    assert np.array_equal(o2.ids, o.ids) and np.array_equal(o2.codes, o.codes)
    assert np.array_equal(o2.tvals, o.tvals)
    g.nprobe = 8; o.nprobe = 8
    D_t, I_t = g.search_dev(torch.from_numpy(xq).cuda(), 10)
    stats = g.last_stats()  # host-side call behind device-stream work
    Do, Io = o.search(xq, 10)
    _assert_same(D_t.cpu().numpy(), I_t.cpu().numpy(), Do, Io, "search_dev")
    assert stats["ndis"] == o.last_ndis
    _assert_same(*g.search(xq, 10), Do, Io, "host search after device search")


# ------------------------------------------------------------------ K1 on tensor cores
@pytest.mark.parametrize("kind,metric,d,M", [("ivf_pq", L2, 128, 32), ("ivf_flat", L2, 64, 0),
                                             ("ivf_flat", IP, 128, 0), ("ivf_sq", L2, 128, 0),
                                             # d = 256: query tile resident for FAST, streamed for PRECISE;
                                             # d = 192 / 768 (config C4's dimension): k-atoms streamed
                                             ("ivf_flat", L2, 256, 0), ("ivf_flat", IP, 192, 0),
                                             ("ivf_sq", L2, 768, 0)])
def test_tensor_core_coarse_quantizer_matches_oracle(kind, metric, d, M):
    """nlist >= 1024 and d a multiple of 64 route the coarse quantizer through wgmma (fp16
    screening: FAST one MMA per k-step, PRECISE hi/lo split, AUTO choosing between them from the
    statistics of the launch before) + canonical fp32 re-rank: probe lists, hence results, must
    still be bit-identical to the oracle's in every mode, and identical to the plain FFMA path."""
    rs = np.random.RandomState(12)
    nlist, n = 1024, _sz(60_000, 6_000)
    g, o, xb = _build_both(kind, metric, d, nlist, M, n, rs, via="gpu")
    xq = np.concatenate([clustered(rs, 150, d, ncl=64), xb[:50] + 0.01 * rs.randn(50, d).astype(np.float32)])
    for nprobe in (1, 7, 64):
        g.nprobe = nprobe; o.nprobe = nprobe
        Do, Io = o.search(xq, 10)
        g.set_param("tensor_cores", 1)
        for mode, name in ((2, "precise"), (1, "fast"), (0, "auto"), (0, "auto, second launch")):
            g.set_param("tc_screen_mode", mode)
            Dg, Ig = g.search(xq, 10)
            _assert_same(Dg, Ig, Do, Io, f"TC coarse ({name}) {kind} nprobe={nprobe}")
            assert g.last_stats()["ndis"] == o.last_ndis
        g.set_param("tensor_cores", 0)
        Df, If = g.search(xq, 10)
        _assert_same(Df, If, Do, Io, f"FFMA coarse {kind} nprobe={nprobe}")
    g.set_param("tensor_cores", 1)
    D1, I1 = g.search(xq[3:4], 10)  # single query: a 128-row tile with one valid row
    g.nprobe = 64
    D1, I1 = g.search(xq[3:4], 10)
    o.nprobe = 64
    _assert_same(D1, I1, *o.search(xq[3:4], 10), "TC coarse nq=1")


def test_tensor_core_near_tie_overflow_is_redone_exactly():
    """More near-tied group minima than the decide stage keeps (duplicate centroids, duplicate
    database rows): the row is flagged (screen_overflow) and tc_exact_rows_kernel redoes it over
    ALL columns, so probe lists / results stay bit-identical to the oracle's -- ids ascending
    among exact ties, and the one populated list among 48 duplicate centroids is still probed."""
    from oracle import oracle as O

    E = _engine()
    rs = np.random.RandomState(21)
    d, nlist = 64, 2048
    # (a) coarse quantizer (search) and assignment (add): 48 copies of one centroid, one per group of 32
    cent = rs.randn(nlist, d).astype(np.float32)
    # (at DEScending positions inside their groups: the packed column index orders equal screening
    # values by position first, so without the exact fallback the LAST copies would be probed)
    cols = 32 * np.arange(48) + (31 - np.arange(48) % 32)
    cent[cols] = cent[cols[0]]
    o = O.make_index("ivf_flat", d, metric=L2, nlist=nlist)
    o.set_state({"centroids": cent, "list_off": np.zeros(nlist + 1, np.int64), "ids": np.zeros(0, np.int64),
                 "vecs": np.zeros((0, d), np.float32)})
    n = _sz(20_000, 3_000)
    xb = (cent[rs.randint(0, nlist, n)] + 0.05 * rs.randn(n, d)).astype(np.float32)
    xb[:200] = cent[cols[0]] + 0.01 * rs.randn(200, d).astype(np.float32)   # rows of the duplicated centroid
    o.add(xb)
    assert np.diff(o.list_off)[cols[1:]].sum() == 0   # ties -> smallest index: only the first copy's list is populated
    g = E.GpuIndex(E.KIND_IVF_FLAT, d, L2, nlist=nlist)
    g.set_state({"centroids": cent, "list_off": np.zeros(nlist + 1, np.int64), "ids": np.zeros(0, np.int64),
                 "vecs": np.zeros((0, d), np.float32)})
    g.add(xb)                                          # dfx_tc_assign: rows of the duplicated centroid overflow (G = 6 < 48)
    st = g.get_state()
    assert np.array_equal(st["list_off"], o.list_off) and np.array_equal(st["ids"], o.ids)
    xq = np.concatenate([cent[cols[0]][None] + 0.01 * rs.randn(40, d), xb[300:340]]).astype(np.float32)
    for nprobe in (1, 4, 20, 40):                      # decide_rows_kernel<0> (all 64 groups kept); 40 > 32: rerank_kernel<2>
        g.nprobe = nprobe; o.nprobe = nprobe
        Do, Io = o.search(xq, 10)
        for mode in (2, 1, 0):
            g.set_param("tc_screen_mode", mode)
            _assert_same(*g.search(xq, 10), Do, Io, f"duplicate centroids nprobe={nprobe} mode={mode}")
            assert g.last_stats()["ndis"] == o.last_ndis
    # (b) flat search: 64 copies of one row spread over 64 groups, k = 10 (G = 18 groups kept)
    for metric in (IP, L2):
        xf = rs.randn(_sz(8192, 4096), d).astype(np.float32)
        fc = 32 * np.arange(64) + (31 - np.arange(64) % 32)
        xf[fc] = xf[fc[0]]
        gf = E.GpuIndex(E.KIND_FLAT, d, metric)
        gf.add(xf)
        qf = np.concatenate([xf[fc[0]][None] * 1.0 + 0.001 * rs.randn(8, d), rs.randn(8, d)]).astype(np.float32)
        Do, Io = O.flat_search(metric, xf, qf, 10)
        for mode in (2, 1, 0):
            gf.set_param("tc_screen_mode", mode)
            _assert_same(*gf.search(qf, 10), Do, Io, f"duplicate rows flat metric={metric} mode={mode}")


def test_tensor_core_many_groups_select_from_all_candidates():
    """nlist 8192 = 256 groups of 32 lists: nprobe 128 keeps G = 136 groups, more candidate slots
    (G x 32 > 4096) than the fused decide kernel sorts in shared memory, so every candidate's exact
    composite is written out (rerank_kernel<0>) and the top-nprobe selected from them; nprobe 1 / 7
    take decide_rows_kernel and 40 rerank_kernel<2>.  Centroids come from set_state (no
    training), rows are assigned by the tensor-core screening (dfx_tc_assign)."""
    from oracle import oracle as O

    E = _engine()
    rs = np.random.RandomState(31)
    d, nlist = 64, 8192
    cent = rs.randn(nlist, d).astype(np.float32)

    def empty():
        return {"centroids": cent, "list_off": np.zeros(nlist + 1, np.int64), "ids": np.zeros(0, np.int64),
                "vecs": np.zeros((0, d), np.float32)}

    o = O.make_index("ivf_flat", d, metric=L2, nlist=nlist)
    o.set_state(empty())
    g = E.GpuIndex(E.KIND_IVF_FLAT, d, L2, nlist=nlist)
    g.set_state(empty())
    n, nq = _sz(10_000, 2_000), _sz(200, 16)
    xb = (cent[rs.randint(0, nlist, n)] + 0.3 * rs.randn(n, d)).astype(np.float32)
    o.add(xb)
    g.add(xb)
    st = g.get_state()
    assert np.array_equal(st["list_off"], o.list_off) and np.array_equal(st["ids"], o.ids)
    xq = (cent[rs.randint(0, nlist, nq)] + 0.3 * rs.randn(nq, d)).astype(np.float32)
    for nprobe in (1, 7, 40, 128):
        g.nprobe = nprobe; o.nprobe = nprobe
        Do, Io = o.search(xq, 10)
        for mode in (2, 1, 0):
            g.set_param("tc_screen_mode", mode)
            _assert_same(*g.search(xq, 10), Do, Io, f"nlist 8192 nprobe={nprobe} mode={mode}")
            assert g.last_stats()["ndis"] == o.last_ndis


def test_tensor_core_auto_precision_follows_the_data():
    """tc_screen_mode 0 (AUTO): a shard starts with the PRECISE screening (fp16 hi/lo split, three
    MMAs) and moves to FAST (one MMA) only after a window of observed rows none of which would
    have overflowed the kept groups under FAST's wider tolerance (an overflowing row costs an exact
    pass over all lists); on data whose norms dwarf the gaps between neighbouring centroids it
    must stay PRECISE.  The rule is checked against the counters the launches report; results are
    the oracle's either way."""
    from oracle import oracle as O

    E = _engine()
    rs = np.random.RandomState(23)
    d, nlist, n = 64, 2560, _sz(40_000, 8_000)    # 80 groups of 32 lists (with <= 64 all are kept: no overflow)
    A = np.linalg.qr(rs.randn(d, 6))[0].astype(np.float32)
    for offset in (0.0, 300.0):
        xb = (rs.randn(n, 6).astype(np.float32) @ A.T + offset).astype(np.float32)
        g = E.GpuIndex(E.KIND_IVF_FLAT, d, L2, nlist=nlist)
        g.set_param("kmeans_niter", _sz(2, 1))
        g.train(xb[: n // 2])
        g.add(xb)
        o = O.make_index("ivf_flat", d, metric=L2, nlist=nlist)
        o.set_state(g.get_state())
        g.nprobe = 8; o.nprobe = 8
        nb = _sz(1024, 64)                                        # rows per launch
        g.set_param("tc_auto_window", 4 * nb)                     # (default: 16 384 rows)
        xq = xb[:nb] + 0.01 * rs.randn(nb, d).astype(np.float32)
        Do, Io = o.search(xq[:64], 10)
        assert g.get_param("tc_fast") == 0.0                      # AUTO starts PRECISE
        g.search(xq[:1], 10)                                      # a single row decides nothing
        assert g.get_param("tc_fast") == 0.0 and g.get_param("tc_stat_rows") == 1.0
        would = g.get_param("tc_stat_fast_would")
        for it in range(3):                                       # 1 + 3 nb rows: the window is not full yet
            Dg, Ig = g.search(xq, 10)
            _assert_same(Dg[:64], Ig[:64], Do, Io, f"auto precision offset={offset} launch {it}")
            assert g.get_param("tc_fast") == 0.0 and g.get_param("tc_stat_rows") == float(nb)
            would += g.get_param("tc_stat_fast_would")
        Dg, Ig = g.search(xq, 10)                                 # fills the window: the decision
        would += g.get_param("tc_stat_fast_would")
        assert g.get_param("tc_fast") == (1.0 if would == 0 else 0.0), (offset, would)
        if offset:
            assert would > 0                                      # norms 2400, gaps ~1: FAST cannot resolve them
        for it in range(2):                                       # whatever the precision now: same bits
            _assert_same(*g.search(xq[:64], 10), Do, Io, f"auto precision offset={offset}, settled {it}")


def test_tensor_core_assign_matches_oracle():
    """add() with nlist >= 1024 assigns through the tensor-core screening + exact arg-min; the
    lists must be those the oracle builds from the same trained state."""
    from oracle import oracle as O

    E = _engine()
    rs = np.random.RandomState(13)
    d, nlist, M, n = 128, 1024, 32, _sz(80_000, 6_000)
    xb = clustered(rs, n, d, ncl=700, sigma=0.5)
    g = E.GpuIndex(E.KIND_IVF_PQ, d, L2, nlist=nlist, pq_m=M)
    g.set_param("kmeans_niter", _sz(6, 2))
    g.train(xb[:_sz(40000, 3000)])
    third = n // 3
    g.add(xb[:third])                       # AUTO: a PRECISE probe chunk, then by its statistics
    g.set_param("tc_screen_mode", 1)
    g.add(xb[third:2 * third])              # FAST
    g.set_param("tc_screen_mode", 2)
    g.add(xb[2 * third:])                   # PRECISE
    st = g.get_state()
    o = O.OracleIVFPQ(d, nlist, M, 8, coarse_metric=L2)
    o.centroids, o.codebooks, o.is_trained = st["centroids"], st["codebooks"], True
    o.add(xb)
    assert np.array_equal(o.list_off, st["list_off"])
    assert np.array_equal(o.ids, st["ids"])
    assert np.array_equal(o.codes, st["codes"])


def test_interleaved_and_row_major_pq_layouts_agree():
    """IVF-PQ, M=32: the block scan with its fused table build (default) and the row-major scan
    (table from pq_prep_kernel) return the same bits as the oracle; export/import/reconstruct work in
    both layouts and across incremental adds."""
    from oracle import oracle as O

    E = _engine()
    rs = np.random.RandomState(14)
    d, nlist, M, n = 128, _sz(48, 12), 32, _sz(30_011, 3_011)   # odd sizes: partial blocks in most lists
    xb = clustered(rs, n, d, ncl=60)
    xq = xb[:37] + 0.01 * rs.randn(37, d).astype(np.float32)
    g = E.GpuIndex(E.KIND_IVF_PQ, d, L2, nlist=nlist, pq_m=M)
    if EMU:
        g.set_param("kmeans_niter", 3)
    g.train(xb[:_sz(8000, 1500)])
    g.add(xb[:_sz(10_000, n // 3)]); g.nprobe = 6
    D0, I0 = g.search(xq, 10)                        # builds the interleaved form
    g.add(xb[_sz(10_000, n // 3):])                  # incremental add on top of it
    o = O.OracleIVFPQ(d, nlist, M, 8, coarse_metric=L2)
    o.set_state(g.get_state())                       # export de-interleaves
    assert o.ntotal == n
    for nprobe, k in ((6, 10), (nlist, 100), (1, 1)):
        g.nprobe = nprobe; o.nprobe = nprobe
        Do, Io = o.search(xq, k)
        g.set_param("interleaved", 1)
        _assert_same(*g.search(xq, k), Do, Io, f"interleaved nprobe={nprobe}")
        ids = np.array([0, 5, n - 1, -1, _sz(12345, n // 2 + 7)], dtype=np.int64)
        R_il = g.reconstruct_rows(ids)
        g.set_param("interleaved", 0)
        _assert_same(*g.search(xq, k), Do, Io, f"row-major nprobe={nprobe}")
        R_rm = g.reconstruct_rows(ids)
        assert np.array_equal(R_il[[0, 1, 2, 4]], R_rm[[0, 1, 2, 4]]) and np.isnan(R_il[3]).all()
        assert np.allclose(R_il[[0, 1, 2, 4]], o.reconstruct_rows(ids)[[0, 1, 2, 4]], rtol=0, atol=1e-6)
    g.set_param("interleaved", 1)
    g2 = E.GpuIndex(E.KIND_IVF_PQ, d, L2, nlist=nlist, pq_m=M)
    g2.set_state(o.get_state())                      # import interleaves
    g2.nprobe = 6; o.nprobe = 6
    _assert_same(*g2.search(xq, 10), *o.search(xq, 10), "imported, interleaved")


def test_block_scan_matches_oracle():
    """IVF-PQ, M=32, the lane-per-vector block scan with the table build fused into its prologue
    (dfx_scan_il2.cu): register top-k (k <= 32) and the shared-memory path (k > 32), one CTA per
    query writing final rows (large batch) and several CTAs per query (small batch) all return the
    oracle's bits, including id ties; incremental adds, export/import and reconstruct; d = 64 and
    d = 256 take the generic-dsub table build."""
    from oracle import oracle as O

    E = _engine()
    rs = np.random.RandomState(21)
    d, nlist, M, n = 128, _sz(48, 12), 32, _sz(30_011, 3_011)
    xb = clustered(rs, n, d, ncl=60)
    xb[-500:] = xb[:500]                             # exact duplicates: ties decided by the id
    xq = xb[:37] + 0.01 * rs.randn(37, d).astype(np.float32)
    xq[:5] = xb[:5]
    g = E.GpuIndex(E.KIND_IVF_PQ, d, L2, nlist=nlist, pq_m=M)
    if EMU:
        g.set_param("kmeans_niter", 3)
    g.train(xb[:_sz(8000, 1500)])
    g.add(xb[:_sz(10_000, n // 3)]); g.nprobe = 6
    g.search(xq, 10)                                 # builds the blocks
    g.add(xb[_sz(10_000, n // 3):])                  # incremental add on top of them
    o = O.OracleIVFPQ(d, nlist, M, 8, coarse_metric=L2)
    o.set_state(g.get_state())
    assert o.ntotal == n
    ids = np.array([0, 5, n - 1, -1, _sz(12345, n // 2 + 7)], dtype=np.int64)
    for nprobe, k in ((6, 10), (nlist, 32), (1, 1), (_sz(17, 7), 7), (nlist, 100), (8, 300)):
        g.nprobe = nprobe; o.nprobe = nprobe
        Do, Io = o.search(xq, k)
        _assert_same(*g.search(xq, k), Do, Io, f"block scan nprobe={nprobe} k={k}")
        R2 = g.reconstruct_rows(ids)
        assert np.isnan(R2[3]).all()
        assert np.allclose(R2[[0, 1, 2, 4]], o.reconstruct_rows(ids)[[0, 1, 2, 4]], rtol=0, atol=1e-6)
    for nq in (1, 3, 200, _sz(1500, 200)):           # one list per CTA ... one CTA per query
        q = np.ascontiguousarray(np.tile(xq, (_sz(41, 6), 1))[:nq])
        g.nprobe = 9; o.nprobe = 9
        _assert_same(*g.search(q, 10), *o.search(q, 10), f"block scan nq={nq}")
    g2 = E.GpuIndex(E.KIND_IVF_PQ, d, L2, nlist=nlist, pq_m=M)
    g2.set_state(o.get_state())
    g2.nprobe = 6; o.nprobe = 6
    _assert_same(*g2.search(xq, 10), *o.search(xq, 10), "imported")
    for d2 in (64, 256):                             # dsub = 2 / 8: generic table build
        xb2 = clustered(rs, _sz(6000, 1500), d2, ncl=40)
        g3 = E.GpuIndex(E.KIND_IVF_PQ, d2, L2, nlist=8, pq_m=32)
        g3.set_param("kmeans_niter", 3)
        g3.train(xb2[:_sz(3000, 1000)]); g3.add(xb2); g3.nprobe = 4
        o3 = O.OracleIVFPQ(d2, 8, 32, 8, coarse_metric=L2)
        o3.set_state(g3.get_state()); o3.nprobe = 4
        for nq in (2, _sz(700, 90)):
            q = np.ascontiguousarray(np.tile(xb2[:50], (_sz(14, 2), 1))[:nq])
            _assert_same(*g3.search(q, 10), *o3.search(q, 10), f"block scan d={d2} nq={nq}")


@pytest.mark.parametrize("metric", [IP, L2])
def test_flat_tensor_core_path_matches_oracle(metric):
    """flat_tensor_cores=1 (the default): screening on tensor cores + exact canonical re-rank returns the bits of
    the plain GEMM path and of the oracle (ties, k up to 100, rows added after the first search)"""
    from oracle import oracle as O

    E = _engine()
    rs = np.random.RandomState(31)
    d, n = 128, _sz(100_000, 5_000)
    xb = clustered(rs, n, d, ncl=200)
    xb[-300:] = xb[:300]                              # exact duplicates: ties decided by the id
    xq = np.concatenate([xb[:20], clustered(rs, 17, d, ncl=200)])
    g = E.GpuIndex(E.KIND_FLAT, d, metric)
    o = O.make_index("flat", d, metric=metric)
    g.add(xb[: n // 2]); o.add(xb[: n // 2])
    for k in (1, 10, 33, 100):
        Do, Io = o.search(xq, k)
        g.set_param("flat_tensor_cores", 1)
        for mode in (2, 1, 0):
            g.set_param("tc_screen_mode", mode)
            _assert_same(*g.search(xq, k), Do, Io, f"flat TC k={k} mode={mode}")
        g.set_param("flat_tensor_cores", 0)
        _assert_same(*g.search(xq, k), Do, Io, f"flat GEMM k={k}")
    g.add(xb[n // 2:]); o.add(xb[n // 2:])            # the fp16 copy must follow
    g.set_param("flat_tensor_cores", 1)
    _assert_same(*g.search(xq, 10), *o.search(xq, 10), "flat TC after add")
    _assert_same(*g.search(xq[:1], 5), *o.search(xq[:1], 5), "flat TC nq=1")


# ------------------------------------------------------------------ exchange kernels of the data plane
class _Dev:
    """a device buffer for the raw `*_dev` entry points: a CUDA tensor on a GPU, the numpy array
    itself on the emulated library (its 'device memory' is host memory)"""

    def __init__(self, arr):
        self.shape, self.dtype = arr.shape, arr.dtype
        if EMU:
            self.a = np.ascontiguousarray(arr).copy()
            self.ptr = self.a.ctypes.data
        else:
            import torch

            self.t = torch.from_numpy(np.ascontiguousarray(arr)).cuda()
            self.ptr = self.t.data_ptr()

    def get(self):
        if EMU:
            return self.a
        import torch

        torch.cuda.synchronize()
        return self.t.cpu().numpy()


def test_exchange_kernels_match_numpy():
    """dfx_merge_packed_dev == dfx_merge over the same blocks (the layout ONE all-gather delivers);
    dfx_encode_ids_dev / dfx_filter_compact_dev == the reference's post-filter loop
    (client.py:229-250); dfx_reconstruct_dev with a shard tag decodes exactly the owned winners"""
    import ctypes as C
    from oracle import oracle as O

    E = _engine()
    L = E.lib()
    rs = np.random.RandomState(77)
    R, S_loc, nq, k = 3, 2, 9, 5
    n = S_loc * nq * k
    D = np.sort(rs.rand(R * S_loc, nq, k).astype(np.float32), axis=2)
    D[1, :, 3:] = np.finfo(np.float32).max                 # a shard with fewer than k hits
    D[2, 4, :] = D[0, 4, :]                                  # exact ties across shards: earlier shard wins
    I = rs.randint(0, 1 << 40, size=(R * S_loc, nq, k)).astype(np.int64)
    I[1, :, 3:] = -1
    off_I = (4 * n + 7) & ~7
    stride = off_I + 8 * n + 8
    packed = np.zeros(R * stride, dtype=np.uint8)
    for r in range(R):
        blk = packed[r * stride:(r + 1) * stride]
        blk[:4 * n] = D[r * S_loc:(r + 1) * S_loc].reshape(-1).view(np.uint8)
        blk[off_I:off_I + 8 * n] = I[r * S_loc:(r + 1) * S_loc].reshape(-1).view(np.uint8)
    for negate in (0, 1):
        Dm = -D if negate else D
        Dm = np.where(np.abs(D) >= np.finfo(np.float32).max, D, Dm).astype(np.float32)
        Dref, Pref = O.merge(Dm, np.arange(I.size, dtype=np.int64).reshape(I.shape))
        Iref = np.where(Pref >= 0, I.reshape(-1)[np.maximum(Pref, 0)], -1)
        src = np.where(np.abs(D) >= np.finfo(np.float32).max, np.float32(-3.4e38) if negate else D, D).astype(np.float32)
        for r in range(R):
            packed[r * stride:r * stride + 4 * n] = src[r * S_loc:(r + 1) * S_loc].reshape(-1).view(np.uint8)
        dp, oD, oI = _Dev(packed), _Dev(np.zeros((nq, k), np.float32)), _Dev(np.zeros((nq, k), np.int64))
        rc = L.dfx_merge_packed_dev(C.c_int64(R), C.c_int64(S_loc), C.c_int64(nq), C.c_int64(k), C.c_void_p(dp.ptr),
                                    C.c_int64(stride), C.c_int64(off_I), C.c_int(negate), C.c_void_p(oD.ptr),
                                    C.c_void_p(oI.ptr), None)
        assert rc == 0, L.dfx_last_error()
        Dh, Ih = E.merge(src, I, negate=bool(negate))       # the unpacked entry point on the same blocks
        assert np.array_equal(oD.get(), Dh) and np.array_equal(oI.get(), Ih)
        if not negate:
            assert np.array_equal(Dh, Dref) and np.array_equal(Ih, Iref)

    # encode + filter: flags ride in bit 62, compaction keeps the order and stops at k_out
    ncol = 500
    col = rs.randint(0, 4, size=ncol).astype(np.int32)
    col[rs.rand(ncol) < 0.1] = -2
    kin, kout = 41, 7
    ids = rs.randint(0, ncol, size=(nq, kin)).astype(np.int64)
    ids[:, 30:] = np.where(rs.rand(nq, kin - 30) < 0.5, -1, ids[:, 30:])
    ids[3, :] = np.nonzero(col == 2)[0][0]                  # a query whose every hit is dropped
    Dv = np.sort(rs.rand(nq, kin).astype(np.float32), axis=1)
    d_ids, d_col, d_enc = _Dev(ids), _Dev(col), _Dev(np.zeros_like(ids))
    assert L.dfx_encode_ids_dev(C.c_int64(ids.size), C.c_void_p(d_ids.ptr), C.c_int64(5), C.c_void_p(d_col.ptr),
                                C.c_int32(2), C.c_void_p(d_enc.ptr), None) == 0
    enc = d_enc.get()
    drop = (col[np.maximum(ids, 0)] == 2) | (col[np.maximum(ids, 0)] == -2)
    want = np.where(ids < 0, -1, (5 << 40) | ids | np.where(drop, 1 << 62, 0))
    assert np.array_equal(enc, want)
    d_D, d_oD, d_oI, d_cnt = _Dev(Dv), _Dev(np.zeros((nq, kout), np.float32)), _Dev(np.zeros((nq, kout), np.int64)), \
        _Dev(np.zeros(nq, np.int32))
    d_enc2 = _Dev(enc)
    assert L.dfx_filter_compact_dev(C.c_int64(nq), C.c_int64(kin), C.c_int64(kout), C.c_void_p(d_D.ptr),
                                    C.c_void_p(d_enc2.ptr), C.c_void_p(d_oD.ptr), C.c_void_p(d_oI.ptr),
                                    C.c_void_p(d_cnt.ptr), None) == 0
    oD, oI, cnt = d_oD.get(), d_oI.get(), d_cnt.get()
    for q in range(nq):
        keep = [j for j in range(kin) if ids[q, j] >= 0 and not drop[q, j]][:kout]
        assert cnt[q] == len(keep)
        assert np.array_equal(oI[q, :len(keep)], enc[q, keep]) and np.array_equal(oD[q, :len(keep)], Dv[q, keep])
        assert (oI[q, len(keep):] == -1).all() and (oD[q, len(keep):] == np.finfo(np.float32).max).all()
    assert cnt[3] == 0

    # owner-decoded winners
    d = 64
    xb = rs.rand(300, d).astype(np.float32)
    g = E.GpuIndex(E.KIND_FLAT, d, IP)
    g.add(xb)
    loc = rs.randint(0, 300, size=20).astype(np.int64)
    tags = rs.randint(0, 3, size=20).astype(np.int64)
    enc = (tags << 40) | loc
    enc[::7] |= 1 << 62                                       # a drop flag does not change the owner
    enc[5] = -1
    out0 = rs.rand(20, d).astype(np.float32)
    d_e, d_o = _Dev(enc), _Dev(out0)
    assert L.dfx_reconstruct_dev(g._h, C.c_int64(20), C.c_void_p(d_e.ptr), C.c_int64(1), C.c_void_p(d_o.ptr), None) == 0
    out = d_o.get()
    own = (tags == 1) & (enc >= 0)
    assert np.array_equal(out[own], xb[loc[own]]) and np.array_equal(out[~own], out0[~own])
