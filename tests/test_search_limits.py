"""Search at its size limits, bit for bit against the C oracle.

Each test sits on a place where the search driver changes code path because of a size: the K6
merge past the 2048-entry sort (the MSB radix select), flat search past k = 100 (the FFMA GEMM with
32 768-row tiles) and past its query chunks, the k-paths of every IVF list scan, the CTA shapes of
the M = 32 block scan, the query chunks of the IVF driver, and nprobe at the tensor-core / FFMA
switch and at 4096.  Batches too large for the oracle are compared on a sample of rows (the edges
of every chunk and random rows), and every sampled row searched alone must give the same bits.

CPU: this file's `gpu` tests (EMU_SUBSET) run against the emulated library."""
import ctypes as C
import os
import platform
import shutil
import subprocess
import sys

import numpy as np
import pytest

from tests.conftest import clustered
from tests import oracle_sq8 as S

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
IP, L2 = 0, 1
FMAX = np.finfo(np.float32).max
EMU = bool(os.environ.get("DFX_EMU_LIB"))

# sizes of the search driver (dfx_search.cu, dfx_tc.cu)
FLAT_NT = 32768                  # rows per flat FFMA tile
FLAT_QC = 1024                   # queries per flat FFMA chunk
PART_BUDGET = 128 << 20          # bytes of partial results one IVF query chunk may hold


def _sz(full, emu):
    return emu if EMU else full


def _engine():
    from distributed_faiss_b200 import engine

    return engine


def _assert_same(Dg, Ig, Do, Io, what):
    if not (np.array_equal(Ig, Io) and np.array_equal(Dg, Do)):
        bad = np.argwhere((Ig != Io) | (Dg != Do))
        q, j = bad[0]
        raise AssertionError(f"{what}: {len(bad)} mismatching slots of {Ig.size}; first at q={q} j={j}: "
                             f"gpu=({Dg[q, j]!r},{Ig[q, j]}) oracle=({Do[q, j]!r},{Io[q, j]})")


def _num_sms():
    if EMU:
        return 132
    import torch

    return torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count


def _choose_group(nq, nprobe):
    """the driver's probes per CTA (dfx_search.cu choose_group)"""
    return int(max(1, min(nq * nprobe // (_num_sms() * 8), nprobe, 16)))


def _ivf_chunk(nq, nprobe, k, nlist, use_tc):
    """queries per chunk of the IVF driver: 8192 (tensor-core coarse) or 32 M / nlist (FFMA), and
    a chunk's partial results (qc x ngroups x k composites) within PART_BUDGET"""
    qc = min(8192, 8192 if use_tc else max(1, (32 << 20) // nlist))
    part_max = PART_BUDGET // 8
    q1 = max(1, part_max // (nprobe * k))
    if qc > q1:
        g1 = _choose_group(q1, nprobe)
        qc = min(qc, max(q1, part_max // (-(-nprobe // g1) * k)))
    return min(qc, nq)


def _sample_rows(nq, chunk, rs, extra=16):
    """the first and last row of every chunk, their neighbours, and `extra` random rows"""
    rows = set(rs.randint(0, nq, extra).tolist())
    for q0 in range(0, nq, chunk):
        q1 = min(nq, q0 + chunk) - 1
        rows |= {q0, q0 + 1, q1 - 1, q1}
    return np.array(sorted(r for r in rows if 0 <= r < nq))


def _check_sample(g, xq, k, D, I, rows, oracle_search, what):
    """rows of a big batch: the oracle's bits, and the same bits when searched alone"""
    Do, Io = oracle_search(xq[rows], k)
    _assert_same(D[rows], I[rows], Do, Io, what)
    for r in rows:
        D1, I1 = g.search(xq[r:r + 1], k)
        _assert_same(D1, I1, D[r:r + 1], I[r:r + 1], f"{what}: row {r} alone")


# ------------------------------------------------------------------ K6 merge on the radix path
MERGE_SHAPES = [(2, 1024), (3, 683), (8, 1024), (5, 4096)]      # S*k = 2048 (sort), 2049, 8192, 20480
MERGE_PATTERNS = ["random", "equal", "top3", "signed_zero", "negative", "padded", "padded_negative"]


def _merge_inputs(pattern, S_, nq, k, rs):
    """D [S, nq, k] as the shards return it, and whether the merge maximises (negate)"""
    shape = (S_, nq, k)
    negate = pattern in ("negative", "padded_negative")
    if pattern == "random":
        D = rs.rand(*shape).astype(np.float32)
        D[0, :, : k // 2] = D[1 % S_, :, : k // 2]                 # cross-shard ties: the earlier shard wins
    elif pattern == "equal":                                       # radix passes down to the secondary key
        D = np.full(shape, 0.75, dtype=np.float32)
    elif pattern == "top3":                                        # keys share their top three bytes
        D = (np.uint32(0x3F800000) | rs.randint(0, 256, size=shape).astype(np.uint32)).view(np.float32)
    elif pattern == "signed_zero":                                 # -0.0 == +0.0: ties broken by position
        D = np.where(rs.rand(*shape) < 0.5, np.float32(0.0), np.float32(-0.0)).astype(np.float32)
        D[rs.rand(*shape) < 0.05] = np.float32(1e-38)
        D[rs.rand(*shape) < 0.02] = np.float32(-1e-38)
    elif pattern == "negative":
        D = -(0.5 + rs.rand(*shape)).astype(np.float32)
        D[-1, :, : k // 3] = D[0, :, : k // 3]
    else:
        D = rs.rand(*shape).astype(np.float32)
        if negate:
            D = -D
        pads = np.array([FMAX, np.inf, np.nan], dtype=np.float32) * (-1 if negate else 1)
        n = S_ * k
        for q in range(nq):
            nvalid = [k // 2, k, 0, k + 1, n][q] if q < 5 else rs.randint(0, n + 1)
            flat = D[:, q, :].reshape(-1)
            invalid = rs.permutation(n)[: n - nvalid]
            flat[invalid] = pads[np.arange(len(invalid)) % 3]
            D[:, q, :] = flat.reshape(S_, k)
    return np.ascontiguousarray(D, dtype=np.float32), negate


@pytest.mark.gpu
@pytest.mark.parametrize("pattern", MERGE_PATTERNS)
@pytest.mark.parametrize("S_,k", MERGE_SHAPES)
def test_merge_at_large_widths_matches_oracle(S_, k, pattern):
    """dfx_merge and dfx_merge_packed_dev against oracle.merge: rows of S*k entries up to 20 480, so
    past the 2048-entry sort every row goes through the radix select"""
    from oracle import oracle as O
    from tests.test_gpu_parity import _Dev

    E = _engine()
    L = E.lib()
    rs = np.random.RandomState(100 + S_ * k)
    nq = _sz(8, 5)
    D, negate = _merge_inputs(pattern, S_, nq, k, rs)
    I = rs.randint(0, 1 << 40, size=D.shape).astype(np.int64)
    outD, outI = E.merge(D, I, negate=negate)
    pos = np.arange(D.size, dtype=np.int64).reshape(D.shape)
    refD, refP = O.merge(-D if negate else D, pos)
    refI = np.where(refP >= 0, I.reshape(-1)[np.maximum(refP, 0)], -1)
    _assert_same(outD, outI, refD, refI, f"merge S={S_} k={k} {pattern}")
    if pattern.startswith("padded"):
        assert (refI[0] == -1).sum() == k - k // 2 and (refI[1] >= 0).all() and (refI[2] == -1).all()
    # the same shards as one all-gather delivers them: R ranks of S_loc shards
    S_loc = 2 if S_ % 2 == 0 else 1
    R = S_ // S_loc
    n_loc = S_loc * nq * k
    off_I = (4 * n_loc + 7) & ~7
    stride = off_I + 8 * n_loc
    packed = np.zeros(R * stride, dtype=np.uint8)
    for r in range(R):
        blk = packed[r * stride:(r + 1) * stride]
        blk[:4 * n_loc] = D[r * S_loc:(r + 1) * S_loc].reshape(-1).view(np.uint8)
        blk[off_I:off_I + 8 * n_loc] = I[r * S_loc:(r + 1) * S_loc].reshape(-1).view(np.uint8)
    dp, oD, oI = _Dev(packed), _Dev(np.zeros((nq, k), np.float32)), _Dev(np.zeros((nq, k), np.int64))
    rc = L.dfx_merge_packed_dev(C.c_int64(R), C.c_int64(S_loc), C.c_int64(nq), C.c_int64(k), C.c_void_p(dp.ptr),
                                C.c_int64(stride), C.c_int64(off_I), C.c_int(int(negate)), C.c_void_p(oD.ptr),
                                C.c_void_p(oI.ptr), None)
    assert rc == 0, L.dfx_last_error()
    _assert_same(oD.get(), oI.get(), refD, refI, f"packed merge R={R} S_loc={S_loc} k={k} {pattern}")


# ------------------------------------------------------------------ flat search past k = 100
FLAT_KS = [101, 1000, 2048, 2049, 4096]


def _flat_data(N, d, rs):
    xb = rs.randn(N, d).astype(np.float32)
    for t in range(1, -(-N // FLAT_NT)):                # exact copies of the first rows in every later
        xb[t * FLAT_NT:] = xb[: N - t * FLAT_NT]          # tile: ties across tiles
    return xb


def _flat_f64(metric, xb, xq, k):
    """float64 restatement: values sorted best first (ids ascending among equal values)"""
    xb64, xq64 = xb.astype(np.float64), xq.astype(np.float64)
    ip = xq64 @ xb64.T
    if metric == IP:
        key = -ip
    else:
        key = (xq64 ** 2).sum(1)[:, None] - 2 * ip + (xb64 ** 2).sum(1)[None, :]
    order = np.argsort(key, axis=1, kind="stable")[:, :k]
    D = np.take_along_axis(key, order, axis=1)
    return (-D if metric == IP else D), order


def _assert_close_f64(metric, xb, xq, k, Dg, Ig, what):
    D64, I64 = _flat_f64(metric, xb, xq, k)
    kk = D64.shape[1]
    scale = (xq.astype(np.float64) ** 2).sum(1, keepdims=True) + (xb.astype(np.float64) ** 2).sum(1).max()
    assert (np.abs(Dg[:, :kk] - D64) <= 1e-4 * scale).all(), what
    gap = np.abs(np.diff(D64, axis=1))
    sep = np.ones_like(I64, dtype=bool)
    sep[:, 1:] &= gap > 1e-5 * scale
    sep[:, :-1] &= gap > 1e-5 * scale
    assert np.array_equal(Ig[:, :kk][sep], I64[sep]), what


@pytest.mark.gpu
@pytest.mark.parametrize("N", [2 * FLAT_NT + 17, 3000])
@pytest.mark.parametrize("metric", [IP, L2])
def test_flat_large_k_matches_oracle(metric, N):
    """k in 101..4096 runs the FFMA GEMM, a select per 32 768-row tile and one over ntiles * k.
    N = 2 tiles + 17 rows: the last tile is shorter than k, ties cross tiles; N = 3000 < k: padding.
    k = 100 (tensor-core screening) is the first 100 columns of k = 101, bit for bit."""
    from oracle import oracle as O

    E = _engine()
    rs = np.random.RandomState(200 + N)
    d = 64
    xb = _flat_data(N, d, rs)
    xq = np.concatenate([xb[[5, 7]], rs.randn(_sz(6, 2), d).astype(np.float32)])   # rows 0, 1: in the database
    g = E.GpuIndex(E.KIND_FLAT, d, metric)
    g.add(xb)
    for k in FLAT_KS:
        Dg, Ig = g.search(xq, k)
        Do, Io = O.flat_search(metric, xb, xq, k)
        _assert_same(Dg, Ig, Do, Io, f"flat metric={metric} N={N} k={k}")
        _assert_close_f64(metric, xb, xq, k, Dg, Ig, f"flat float64 metric={metric} N={N} k={k}")
        if k > N:
            assert (Ig[:, N:] == -1).all() and (Dg[:, N:] == (-FMAX if metric == IP else FMAX)).all()
        if metric == L2:
            assert Dg[0, 0] >= 0 and Ig[0, 0] == 5         # ||q - x||^2 clamped at 0, the smallest id first
        if metric == L2 and N > FLAT_NT:                   # the copies in the next tiles follow, by id
            assert Ig[0, :3].tolist() == [5, 5 + FLAT_NT, 5 + 2 * FLAT_NT]
            assert Dg[0, 0] == Dg[0, 1] == Dg[0, 2]
        if k == 101:
            D100, I100 = g.search(xq, 100)                 # tensor-core screening + exact re-rank
            _assert_same(D100, I100, Dg[:, :100], Ig[:, :100], f"flat TC k=100 vs FFMA k=101 N={N}")


@pytest.mark.gpu
@pytest.mark.parametrize("metric", [IP, L2])
def test_flat_query_chunks_match_oracle(metric):
    """batches across the FFMA path's 1024-query chunks (k > 100) and across the tensor-core path's
    QT-query chunks (k <= 100), compared on the rows at every chunk edge"""
    from oracle import oracle as O

    E = _engine()
    rs = np.random.RandomState(300 + metric)
    d, N = 64, 2 * FLAT_NT + 17
    xb = _flat_data(N, d, rs)
    g = E.GpuIndex(E.KIND_FLAT, d, metric)
    g.add(xb)

    def oracle_search(q, k):
        return O.flat_search(metric, xb, q, k)

    for nq, k in ((FLAT_QC - 1, 101), (FLAT_QC + 1, 2049), (2 * FLAT_QC + 5, 101), (2 * FLAT_QC + 5, 4096)):
        xq = rs.randn(nq, d).astype(np.float32)
        xq[min(FLAT_QC, nq - 1)] = xb[11]                  # the first row of the second chunk is a database row
        D, I = g.search(xq, k)
        rows = _sample_rows(nq, FLAT_QC, rs, extra=_sz(16, 4))
        _check_sample(g, xq, k, D, I, rows, oracle_search, f"flat FFMA chunks nq={nq} k={k}")
    ng = -(-N // 128) * 4
    QT = max(128, ((64 << 20) // (ng * 4)) // 128 * 128)   # queries per tensor-core chunk
    nq = QT + 37
    xq = rs.randn(nq, d).astype(np.float32)
    xq[QT] = xb[12]
    for k in (10, 100):
        D, I = g.search(xq, k)
        rows = _sample_rows(nq, QT, rs, extra=_sz(16, 4))
        _check_sample(g, xq, k, D, I, rows, oracle_search, f"flat TC chunks nq={nq} k={k}")


# ------------------------------------------------------------------ IVF: the k-paths of every list scan
IVF_KS = [32, 33, 128, 129, 512, 513, 1024]
IVF_KINDS = {
    "ivf_flat_ip": ("ivf_flat", IP, 64, 0, None),
    "ivf_flat_l2": ("ivf_flat", L2, 64, 0, None),
    "ivf_sq": ("ivf_sq", L2, 64, 0, None),
    "ivf_sq8": ("ivf_sq8", L2, 64, 0, None),
    "pq16": ("ivf_pq", L2, 64, 16, None),
    "pq24": ("ivf_pq", L2, 96, 24, None),
    "pq64": ("ivf_pq", L2, 128, 64, None),
    "pq32_interleaved": ("ivf_pq", L2, 128, 32, 1),
    "pq32_row_major": ("ivf_pq", L2, 128, 32, 0),
}


def _ivf_pair(kind, metric, d, nlist, M, n, rs, ncl):
    """a shard trained and filled on the GPU, and the oracle holding the same shard"""
    E = _engine()
    kinds = {"ivf_flat": E.KIND_IVF_FLAT, "ivf_pq": E.KIND_IVF_PQ, "ivf_sq": E.KIND_IVF_SQ16,
             "ivf_sq8": E.KIND_IVF_SQ8}
    xb = clustered(rs, n, d, ncl=ncl)
    g = E.GpuIndex(kinds[kind], d, metric, nlist=nlist, pq_m=M)
    g.set_param("kmeans_niter", _sz(6, 2))
    g.train(xb[: n // 2])
    g.add(xb)
    o = S.make_index(kind, d, metric=metric, nlist=nlist, M=M)
    o.set_state(g.get_state())
    assert g.ntotal == n == o.ntotal
    return g, o, xb


def _ivf_from_centroids(kind, metric, cent, xb, M=0):
    """a shard with the given centroids (no training), rows assigned on the GPU; the oracle copy"""
    E = _engine()
    kinds = {"ivf_flat": E.KIND_IVF_FLAT}
    nlist, d = cent.shape
    st = {"centroids": cent, "list_off": np.zeros(nlist + 1, np.int64), "ids": np.zeros(0, np.int64),
          "vecs": np.zeros((0, d), np.float32)}
    g = E.GpuIndex(kinds[kind], d, metric, nlist=nlist)
    g.set_state(st)
    g.add(xb)
    o = S.make_index(kind, d, metric=metric, nlist=nlist)
    o.set_state(g.get_state())
    return g, o


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(IVF_KINDS))
def test_ivf_k_paths_match_oracle(name):
    """k on both sides of 32, 128 and 512 and at 1024 for every list scan: register / shared-memory
    top-k, the per-CTA merge, padding when fewer than k vectors are probed, one CTA per query
    (ngroups = 1, large batch) and several (small batch)"""
    kind, metric, d, M, il = IVF_KINDS[name]
    rs = np.random.RandomState(400 + list(IVF_KINDS).index(name))
    nlist = _sz(16, 4)
    g, o, xb = _ivf_pair(kind, metric, d, nlist, M, _sz(12_000, 2_400), rs, ncl=4 * nlist)
    if il is not None:
        g.set_param("interleaved", il)
    assert o.ntotal >= 2 * 1024
    # the last query sits on the centroid of the shortest list: padded at nprobe = 1
    xq = np.concatenate([clustered(rs, _sz(5, 3), d, ncl=8), xb[:1], o.centroids[np.argmin(np.diff(o.list_off))][None]])
    for nprobe in (1, 4, nlist):
        g.nprobe = nprobe; o.nprobe = nprobe
        for k in IVF_KS:
            Dg, Ig = g.search(xq, k)
            Do, Io = o.search(xq, k)
            _assert_same(Dg, Ig, Do, Io, f"{name} nprobe={nprobe} k={k}")
            assert g.last_stats()["ndis"] == o.last_ndis
        if nprobe == 1:
            assert (Ig[:, -1] == -1).any()                 # k = 1024 > the probed list: padded
        else:
            assert (Ig[:, -1] >= 0).any()                  # k = 1024 < the probed vectors: filled
        if nprobe == nlist:
            assert (Ig >= 0).all()
    if EMU:
        return
    nq = 1100                                              # choose_group: one CTA per query at nprobe 4
    assert -(-4 // _choose_group(nq, 4)) == 1
    xq = clustered(rs, nq, d, ncl=16)
    g.nprobe = 4; o.nprobe = 4
    for k in IVF_KS:
        Dg, Ig = g.search(xq, k)
        _assert_same(Dg, Ig, *o.search(xq, k), f"{name} nq={nq} nprobe=4 k={k}")


# ------------------------------------------------------------------ the M = 32 block scan's CTA shapes
@pytest.mark.gpu
@pytest.mark.parametrize("threads", [256, 512])
def test_block_scan_shapes_match_oracle(threads):
    """il2_threads x il2_prefetch x k: every CTA shape of scan_pq_il2_kernel returns the oracle's
    bits; 512 threads at k > 512 (no room for 16 candidate buffers) runs the 256-thread shape"""
    rs = np.random.RandomState(500)
    nlist = _sz(16, 4)
    g, o, xb = _ivf_pair("ivf_pq", L2, 128, nlist, 32, _sz(8000, 2000), rs, ncl=4 * nlist)
    xq = np.concatenate([clustered(rs, _sz(19, 4), 128, ncl=8), xb[:1]])
    g.set_param("il2_threads", threads)
    assert g.get_param("il2_threads") == threads
    g.nprobe = o.nprobe = _sz(6, 3)
    for k in _sz([1, 10, 32, 33, 300, 1024], [1, 33, 1024]):
        Do, Io = o.search(xq, k)
        for pf in _sz([0, 1, 4, 32], [0, 32]):
            g.set_param("il2_prefetch", pf)
            _assert_same(*g.search(xq, k), Do, Io, f"il2 threads={threads} prefetch={pf} k={k}")
    g.set_param("il2_prefetch", -1)


# ------------------------------------------------------------------ query chunks of the IVF driver
def _probe_ndis(o, cent, metric, xq, nprobe):
    """vectors the probe lists of the oracle's coarse quantizer hold, per query"""
    from oracle import oracle as O

    keys, _ = O.coarse(metric, cent, xq, nprobe)
    lens = np.diff(o.list_off)
    return lens[keys].sum(1)


def _check_chunked(g, o, cent, metric, xq, k, chunk, rs, what, full_ndis=True):
    nprobe = g.nprobe
    D, I = g.search(xq, k)
    ndis = g.last_stats()["ndis"]
    rows = _sample_rows(len(xq), chunk, rs)
    _check_sample(g, xq, k, D, I, rows, o.search, what)
    per_row = _probe_ndis(o, cent, metric, xq[rows], nprobe)
    for r, want in zip(rows, per_row):                      # each sampled row's probe lists
        g.search(xq[r:r + 1], k)
        assert g.last_stats()["ndis"] == want, f"{what}: probe lists of row {r}"
    if full_ndis:
        assert ndis == _probe_ndis(o, cent, metric, xq, nprobe).sum(), f"{what}: ndis"
    return D, I


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["ivf_flat", "ivf_pq"])
def test_ivf_tc_coarse_query_chunks(kind):
    """tensor-core coarse path, 8192 queries per chunk: a batch of 8192 + 37 queries; IVF-PQ M = 32
    with k <= 32 writes its final rows from the scan kernel (one CTA per query)"""
    if EMU:
        pytest.skip("8 k queries: too large for the emulator")
    rs = np.random.RandomState(600)
    nlist, d = 1024, 128 if kind == "ivf_pq" else 64
    g, o, xb = _ivf_pair(kind, L2, d, nlist, 32 if kind == "ivf_pq" else 0, 60_000, rs, ncl=512)
    cent = o.centroids
    nq = 8192 + 37
    xq = xb[rs.randint(0, len(xb), nq)] + 0.05 * rs.randn(nq, d).astype(np.float32)
    g.nprobe = o.nprobe = 8
    assert _ivf_chunk(nq, 8, 10, nlist, True) == 8192
    _check_chunked(g, o, cent, L2, xq, 10, 8192, rs, f"{kind} TC coarse k=10")
    # the bench shape keeps one chunk of 8192 queries: one group per query, 8192 x 10 composites
    assert g.get_param("workspace_bytes") == 8192 * 1 * 10 * 8
    if kind == "ivf_pq":
        _check_chunked(g, o, cent, L2, xq, 32, 8192, rs, "ivf_pq TC coarse k=32", full_ndis=False)


@pytest.mark.gpu
def test_ivf_ffma_coarse_query_chunks():
    """FFMA coarse path (tensor_cores = 0), nlist 65 536: 32 M / nlist = 512 queries per chunk,
    1100 queries make three chunks"""
    rs = np.random.RandomState(700)
    d, nlist = 32, _sz(65_536, 4096)
    cent = rs.randn(nlist, d).astype(np.float32)
    xb = (cent[rs.randint(0, nlist, _sz(131_072, 8192))] + 0.3 * rs.randn(_sz(131_072, 8192), d)).astype(np.float32)
    g, o = _ivf_from_centroids("ivf_flat", L2, cent, xb)
    g.set_param("tensor_cores", 0)
    nq = _sz(1100, 20)
    chunk = _ivf_chunk(nq, 16, 10, nlist, False)
    assert EMU or chunk == 512
    xq = (cent[rs.randint(0, nlist, nq)] + 0.3 * rs.randn(nq, d)).astype(np.float32)
    g.nprobe = o.nprobe = 16
    _check_chunked(g, o, cent, L2, xq, 10, chunk, rs, "FFMA coarse chunks")


@pytest.mark.gpu
def test_ivf_tc_coarse_inner_chunks():
    """nlist 131 072 at d = 64: the tensor-core coarse call splits a batch into 64 M / (ng * 4) =
    4096-query chunks of its own (its statistics come from the last one)"""
    if EMU:
        pytest.skip("131 072 lists: too large for the emulator")
    rs = np.random.RandomState(800)
    d, nlist = 64, 131_072
    cent = rs.randn(nlist, d).astype(np.float32)
    n = 262_144
    xb = (cent[rs.randint(0, nlist, n)] + 0.3 * rs.randn(n, d)).astype(np.float32)
    g, o = _ivf_from_centroids("ivf_flat", L2, cent, xb)
    ng = nlist // 32
    inner = max(128, ((64 << 20) // (ng * 4)) // 128 * 128)
    assert inner == 4096
    nq = inner + 37
    xq = (cent[rs.randint(0, nlist, nq)] + 0.3 * rs.randn(nq, d)).astype(np.float32)
    g.nprobe = o.nprobe = 8
    _check_chunked(g, o, cent, L2, xq, 10, inner, rs, "TC coarse inner chunks", full_ndis=False)


# ------------------------------------------------------------------ nprobe limits
@pytest.mark.gpu
def test_nprobe_at_the_tc_ffma_switch():
    """nprobe 512 takes the tensor-core coarse path, 513 the FFMA one; both, and FFMA at 512, give
    the oracle's bits"""
    rs = np.random.RandomState(900)
    d, nlist = 64, 1024
    cent = rs.randn(nlist, d).astype(np.float32)
    n = _sz(60_000, 6_000)
    xb = (cent[rs.randint(0, nlist, n)] + 0.3 * rs.randn(n, d)).astype(np.float32)
    g, o = _ivf_from_centroids("ivf_flat", L2, cent, xb)
    xq = (cent[rs.randint(0, nlist, _sz(40, 4))] + 0.3 * rs.randn(_sz(40, 4), d)).astype(np.float32)
    for nprobe in (512, 513):
        g.nprobe = o.nprobe = nprobe
        for k in (10, 100):
            Do, Io = o.search(xq, k)
            for tc in (1, 0):
                g.set_param("tensor_cores", tc)
                _assert_same(*g.search(xq, k), Do, Io, f"nprobe={nprobe} k={k} tensor_cores={tc}")
                assert g.last_stats()["ndis"] == o.last_ndis


@pytest.mark.gpu
def test_full_probe_at_k1024_stays_within_the_workspace():
    """nprobe = nlist = 4096 with k = 1024: each query reduces ngroups x 1024 composites (radix
    select); the query chunk keeps the partial results within 128 MiB however large the batch"""
    rs = np.random.RandomState(1000)
    d, nlist, k = 32, 4096, 1024
    cent = rs.randn(nlist, d).astype(np.float32)
    n = _sz(40_000, 6_000)
    xb = (cent[rs.randint(0, nlist, n)] + 0.3 * rs.randn(n, d)).astype(np.float32)
    g, o = _ivf_from_centroids("ivf_flat", L2, cent, xb)
    g.nprobe = o.nprobe = nlist
    xq = (cent[rs.randint(0, nlist, 16)] + 0.3 * rs.randn(16, d)).astype(np.float32)
    Dg, Ig = g.search(xq, k)
    _assert_same(Dg, Ig, *o.search(xq, k), "nprobe=nlist=4096 k=1024 nq=16")
    assert g.last_stats()["ndis"] == 16 * n and (Ig >= 0).all()
    assert g.get_param("workspace_bytes") <= PART_BUDGET
    if EMU:
        return
    nq = 8192
    chunk = _ivf_chunk(nq, nlist, k, nlist, False)
    assert chunk < nq
    xq = (cent[rs.randint(0, nlist, nq)] + 0.3 * rs.randn(nq, d)).astype(np.float32)
    D, I = g.search(xq, k)
    assert g.last_stats()["ndis"] == nq * n
    assert g.get_param("workspace_bytes") <= PART_BUDGET
    rows = _sample_rows(nq, chunk, rs)
    _check_sample(g, xq, k, D, I, rows, o.search, f"nprobe=nlist=4096 k=1024 nq={nq}")


# ------------------------------------------------------------------ the gpu tests on the emulator
EMU_SUBSET = [
    "tests/test_search_limits.py::test_merge_at_large_widths_matches_oracle",
    "tests/test_search_limits.py::test_flat_large_k_matches_oracle[1-3000]",
    "tests/test_search_limits.py::test_ivf_k_paths_match_oracle[ivf_flat_l2]",
    "tests/test_search_limits.py::test_ivf_k_paths_match_oracle[ivf_sq8]",
    "tests/test_search_limits.py::test_ivf_k_paths_match_oracle[pq16]",
    "tests/test_search_limits.py::test_ivf_k_paths_match_oracle[pq32_interleaved]",
    "tests/test_search_limits.py::test_block_scan_shapes_match_oracle",
    "tests/test_search_limits.py::test_full_probe_at_k1024_stays_within_the_workspace",
]
EMU_COUNT = len(MERGE_SHAPES) * len(MERGE_PATTERNS) + 1 + 4 + 2 + 1


def test_search_limits_gpu_tests_on_the_emulated_library():
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
    assert f"{EMU_COUNT} passed" in run.stdout, tail
