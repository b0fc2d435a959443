"""IVF-SQ8 (faiss IndexIVFScalarQuantizer QT_8bit, the factory string "IVF{n},SQ8").

CPU: the oracle (tests/oracle_sq8.py) on known answers and against the float64 restatement, the
faiss file format, and this file's `gpu` tests run against the emulated library.
GPU: the CUDA kernels against the oracle, bit for bit (distances, ids, ndis, trained vector, codes,
reconstruction)."""
import os
import platform
import shutil
import struct
import subprocess
import sys
from fractions import Fraction

import numpy as np
import pytest

from tests.conftest import clustered
from tests import oracle_sq8 as S

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
IP, L2 = 0, 1
FMAX = np.finfo(np.float32).max
EMU = bool(os.environ.get("DFX_EMU_LIB"))


def _sz(full, emu):
    return emu if EMU else full


# ------------------------------------------------------------------ oracle, CPU
def test_fma32_is_correctly_rounded():
    rs = np.random.RandomState(0)
    a = (rs.randn(4000) * 10.0 ** rs.randint(-6, 6, 4000)).astype(np.float32)
    b = (rs.randn(4000) * 10.0 ** rs.randint(-6, 6, 4000)).astype(np.float32)
    c = (-(a.astype(np.float64) * b) * (1 + 1e-7 * rs.randn(4000))).astype(np.float32)  # heavy cancellation
    c[::3] = rs.randn(len(c[::3])).astype(np.float32)
    r = S.fma32(a, b, c)
    for ai, bi, ci, ri in zip(a[:1500], b[:1500], c[:1500], r[:1500]):
        exact = Fraction(float(ai)) * Fraction(float(bi)) + Fraction(float(ci))
        err = abs(Fraction(float(ri)) - exact)
        for nb in (np.nextafter(ri, np.float32(np.inf)), np.nextafter(ri, np.float32(-np.inf))):
            e2 = abs(Fraction(float(nb)) - exact)
            assert err < e2 or (err == e2 and (int(ri.view(np.uint32)) & 1) == 0), (ai, bi, ci, ri)


def test_sq8_codec_known_answers():
    d = 8
    vmin = np.array([1.5, -2, 0, 0, -1, 3, 0.25, 7], dtype=np.float32)
    vdiff = np.array([0, 4, 1, 2, 2, 0, 0.5, 1], dtype=np.float32)   # dims 0 and 5: constant
    tr = np.stack([vmin, vdiff])
    r = np.array([[1.5, -2, 0, 2, 1, 3, 0.75, 8],        # every dim at its minimum / maximum
                  [9.0, -3, -5, 7, 5, -4, 0.5, 7.5],      # outside the range: clamped
                  [0.0, 0, 0.5, 1, 0, 3, 0.5, 7.25]], dtype=np.float32)
    codes = S.sq8_encode_residuals(tr, r)
    assert codes[0].tolist() == [0, 0, 0, 255, 255, 0, 255, 255]
    assert codes[1].tolist() == [0, 0, 0, 255, 255, 0, 127, 127]
    assert codes[2].tolist() == [0, 127, 127, 127, 127, 0, 127, 63]
    dec = S.sq8_decode(tr, codes)
    assert np.array_equal(dec[:, 0], np.full(3, 1.5, np.float32))    # vdiff = 0: decode = vmin
    assert np.array_equal(dec[:, 5], np.full(3, 3.0, np.float32))
    t255 = S.fma32(np.float32(255), S.SQ8_SCALE, S.SQ8_BIAS)
    assert t255 > 1 and np.isclose(t255, 255.5 / 255)                 # code 255 decodes past vmax by half a step
    assert np.array_equal(dec[0, 1], S.fma32(S.fma32(np.float32(0), S.SQ8_SCALE, S.SQ8_BIAS), np.float32(4), np.float32(-2)))


def test_sq8_oracle_search_ties_and_padding():
    d, nlist = 16, 4
    rs = np.random.RandomState(1)
    xb = clustered(rs, 400, d, ncl=4, sigma=0.05)
    xb[:, 3] = 0.25                                   # a constant dimension: vdiff 0 -> code 0
    xb[10:20] = xb[0]                                 # exact duplicates -> exact ties, broken by id
    o = S.make_index("ivf_sq8", d, metric=L2, nlist=nlist)
    o.train(xb)
    o.add(xb[:60])
    assert (o.sq_trained[1, 3] == 0) and (o.codes8[:, 3] == 0).all()
    o.nprobe = 1
    D, I = o.search(xb[:3], 80)                       # k > hits: (FLT_MAX, -1) padding
    assert (I == -1).any() and (D[I == -1] == FMAX).all()
    row = I[0][I[0] >= 0]
    dup = [i for i in range(10, 20)] + [0]
    pos = [list(row).index(i) for i in sorted(dup)]
    assert pos == sorted(pos) and np.all(D[0][pos] == D[0][pos[0]])   # equal distances, ascending ids


@pytest.mark.parametrize("d,nlist", [(32, 8), (64, 16)])
def test_sq8_oracle_close_to_float64(oracle_lib, d, nlist):
    rs = np.random.RandomState(2)
    xb = clustered(rs, 3000, d, ncl=nlist)
    o = S.make_index("ivf_sq8", d, metric=L2, nlist=nlist)
    o.train(xb[:1500]); o.add(xb)
    xq = clustered(rs, 16, d, ncl=8)
    for nprobe in (nlist, 3):
        o.nprobe = nprobe
        Do, Io = o.search(xq, 10)
        D64, I64 = S.ivf_sq8_search_f64(o.get_state(), xq, nprobe, 10)
        scale = (xq.astype(np.float64) ** 2).sum(1, keepdims=True) + (xb.astype(np.float64) ** 2).sum(1).max()
        assert (np.abs(Do - D64) <= 1e-4 * scale).all()
        gap = np.abs(np.diff(D64, axis=1))
        sep = np.ones_like(Io, dtype=bool)
        sep[:, 1:] &= gap > 1e-5 * scale
        sep[:, :-1] &= gap > 1e-5 * scale
        assert np.array_equal(Io[sep], I64[sep])


def test_sq8_faiss_file_roundtrip_and_layout(tmp_path):
    from distributed_faiss_b200 import faiss_io

    rs = np.random.RandomState(3)
    d, nlist = 32, 4
    o = S.make_index("ivf_sq8", d, metric=IP, nlist=nlist)
    xb = clustered(rs, 300, d, ncl=4)
    o.train(xb); o.add(xb)
    st = o.get_state()
    path = str(tmp_path / "sq8.faiss")
    faiss_io.write_index(st, path, nprobe=3)
    st2, nprobe = faiss_io.read_index(path)
    assert nprobe == 3 and st2["kind"] == "ivf_sq8" and st2["coarse_metric"] == IP
    for key in ("centroids", "sq_trained", "list_off", "ids", "codes8"):
        assert np.asarray(st2[key]).tobytes() == np.asarray(st[key]).tobytes(), key
    raw = open(path, "rb").read()
    assert raw[:4] == b"IwSq"
    assert struct.unpack_from("<iqqqBi", raw, 4) == (32, 300, 1 << 20, 1 << 20, 1, 1)   # the index is L2
    off = 4 + 33
    assert struct.unpack_from("<QQ", raw, off) == (4, 3)
    off += 16
    assert raw[off:off + 4] == b"IxFI"                                  # IP coarse quantizer
    off += 4 + 33 + 8 + 4 * 32 * 4 + 9
    assert struct.unpack_from("<iif", raw, off) == (0, 0, 0.0)          # QT_8bit, RS_minmax, arg 0
    off += 12
    assert struct.unpack_from("<QQQ", raw, off) == (32, 32, 64)         # sq.d, sq.code_size, 2d trained
    off += 24
    assert raw[off:off + 256] == st["sq_trained"].astype("<f4").tobytes()   # [vmin, vdiff]
    off += 256
    assert struct.unpack_from("<QB", raw, off) == (32, 1)               # code_size, by_residual
    off += 9
    assert raw[off:off + 4] == b"ilar" and struct.unpack_from("<QQ", raw, off + 4) == (4, 32)
    assert len(raw) == off + 24 + 40 + 300 * (32 + 8)


def test_sq8_and_fp16_files_are_not_interchangeable(tmp_path):
    from distributed_faiss_b200 import faiss_io
    from distributed_faiss_b200.index import Index
    from distributed_faiss_b200.index_cfg import IndexCfg
    import json
    import pickle

    rs = np.random.RandomState(4)
    d = 16
    o = S.make_index("ivf_sq", d, metric=L2, nlist=4)
    xb = clustered(rs, 200, d, ncl=4)
    o.train(xb); o.add(xb)
    faiss_io.write_index(o.get_state(), str(tmp_path / "index.faiss"))
    pickle.dump(list(range(200)), open(tmp_path / "meta.pkl", "wb"))
    cfg = IndexCfg(faiss_factory="IVF4,SQ8", dim=d, centroids=4, metric="l2")
    open(tmp_path / "cfg.json", "w").write(cfg.to_json_string())
    with pytest.raises(RuntimeError, match="'ivf_sq' but the cfg builds 'ivf_sq8'"):
        Index.from_storage_dir(str(tmp_path), engine_factory=S.oracle_engine_factory)
    assert json.load(open(tmp_path / "cfg.json"))["faiss_factory"] == "IVF4,SQ8"


# ------------------------------------------------------------------ the gpu tests on the emulator
EMU_SUBSET = [
    "tests/test_ivf_sq8.py::test_sq8_matches_oracle[gpu-64]",
    "tests/test_ivf_sq8.py::test_sq8_matches_oracle[oracle-64]",
    "tests/test_ivf_sq8.py::test_sq8_edge_cases",
    "tests/test_ivf_sq8.py::test_sq8_training_and_encoding_match_oracle[1]",
    "tests/test_ivf_sq8.py::test_sq8_reconstruct_matches_oracle",
    "tests/test_ivf_sq8.py::test_sq8_rows_inflight_variants_agree",
]


def test_sq8_gpu_tests_on_the_emulated_library():
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
def _gpu(d, nlist, metric=L2):
    from distributed_faiss_b200 import engine as E

    return E.GpuIndex(E.KIND_IVF_SQ8, d, metric, nlist=nlist)


def _assert_same(Dg, Ig, Do, Io, what):
    if not (np.array_equal(Ig, Io) and np.array_equal(Dg, Do)):
        bad = np.argwhere((Ig != Io) | (Dg != Do))
        q, j = bad[0]
        raise AssertionError(f"{what}: {len(bad)} mismatching slots of {Ig.size}; first at q={q} j={j}: "
                             f"gpu=({Dg[q, j]!r},{Ig[q, j]}) oracle=({Do[q, j]!r},{Io[q, j]})")


def _build_both(d, nlist, n, rs, via, metric=L2):
    xb = clustered(rs, n, d, ncl=max(8, nlist // 2))
    g = _gpu(d, nlist, metric)
    o = S.make_index("ivf_sq8", d, metric=metric, nlist=nlist)
    if via == "gpu":
        if EMU:
            g.set_param("kmeans_niter", 2)
        g.train(xb[: n // 2])
        g.add(xb[: n // 3]); g.add(xb[n // 3:])
        o.set_state(g.get_state())
    else:
        o.train(xb[: n // 2])
        o.add(xb)
        g.set_state(o.get_state())
    assert g.ntotal == n == o.ntotal
    return g, o, xb


@pytest.mark.gpu
@pytest.mark.parametrize("d", [64, 768])
@pytest.mark.parametrize("via", ["gpu", "oracle"])
def test_sq8_matches_oracle(d, via):
    rs = np.random.RandomState(10)
    nlist = 16 if d == 64 else 8
    g, o, xb = _build_both(d, nlist, _sz(6000, 1500), rs, via)
    xq = np.concatenate([clustered(rs, 20, d, ncl=8), xb[:5] + 0.01 * rs.randn(5, d).astype(np.float32)])
    for nprobe in (nlist, 1, 5):
        g.nprobe = nprobe; o.nprobe = nprobe
        for k in (10, 1, 100, 300):
            Dg, Ig = g.search(xq, k)
            Do, Io = o.search(xq, k)
            _assert_same(Dg, Ig, Do, Io, f"ivf_sq8 d={d} via={via} nprobe={nprobe} k={k}")
        assert g.last_stats()["ndis"] == o.last_ndis


@pytest.mark.gpu
def test_sq8_edge_cases():
    """k > hits, empty lists, nprobe > nlist, exact ties, a constant dimension"""
    rs = np.random.RandomState(11)
    d, nlist = 32, 8
    xb = clustered(rs, 600, d, ncl=4, sigma=0.05)
    xb[10:20] = xb[0]
    xb[:, 5] = -0.5
    o = S.make_index("ivf_sq8", d, metric=L2, nlist=nlist)
    o.train(xb); o.add(xb[:37])
    g = _gpu(d, nlist)
    g.set_state(o.get_state())
    assert np.array_equal(g.get_array("sq_trained").reshape(2, d), o.sq_trained)
    for nprobe in (1, 3, 50):
        g.nprobe = nprobe; o.nprobe = nprobe
        Dg, Ig = g.search(xb[:9], 64)
        Do, Io = o.search(xb[:9], 64)
        _assert_same(Dg, Ig, Do, Io, f"edge nprobe={nprobe}")
        assert (Ig == -1).any() and (Dg[Ig == -1] == FMAX).all()
        assert g.last_stats()["ndis"] == o.last_ndis


@pytest.mark.gpu
@pytest.mark.parametrize("metric", [IP, L2])
def test_sq8_training_and_encoding_match_oracle(metric):
    """same centroids, same training rows -> the same [vmin, vdiff] and codes, byte for byte"""
    from oracle import oracle as O

    rs = np.random.RandomState(12)
    d, nlist, n = 64, 16, _sz(4000, 1200)          # n <= 256 nlist: the k-means sample is x itself
    x = clustered(rs, n, d, ncl=8)
    g = _gpu(d, nlist, metric)
    if EMU:
        g.set_param("kmeans_niter", 2)
    g.train(x)
    g.add(x)
    st = g.get_state()
    tr = S.sq8_train(st["centroids"], x, metric)
    assert st["sq_trained"].tobytes() == tr.tobytes()
    lists = O.assign(metric, st["centroids"], x)
    order = np.argsort(lists, kind="stable")
    assert np.array_equal(st["ids"], order)
    assert st["codes8"].tobytes() == S.sq8_encode(tr, st["centroids"], lists, x)[order].tobytes()


@pytest.mark.gpu
def test_sq8_training_uses_the_first_100k_rows():
    from oracle import oracle as O

    if EMU:
        pytest.skip("too large for the emulator")
    rs = np.random.RandomState(13)
    d, nlist, n = 64, 1024, 150_000                # 256 nlist > n: the sample is x; 100 k rows train SQ
    x = clustered(rs, n, d, ncl=256)
    x[120_000:, 0] += 50.0                         # rows past the prefix must not widen the range
    g = _gpu(d, nlist)
    g.set_param("kmeans_niter", 2)
    g.train(x)
    cent = g.get_centroids()
    tr = S.sq8_train(cent, x, L2)
    assert g.get_array("sq_trained").tobytes() == tr.tobytes()
    assert O.assign(L2, cent, x[:1]).shape == (1,)


@pytest.mark.gpu
def test_sq8_reconstruct_matches_oracle():
    rs = np.random.RandomState(14)
    g, o, xb = _build_both(64, 16, _sz(3000, 1000), rs, "oracle")
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
def test_sq8_rows_inflight_variants_agree():
    rs = np.random.RandomState(15)
    g, o, xb = _build_both(128, 8, _sz(4000, 1200), rs, "oracle")
    xq = clustered(rs, 12, 128, ncl=8)
    g.nprobe = 3
    out = {}
    for u in (4, 8):
        g.set_param("rows_inflight", u)
        out[u] = g.search(xq, 20)
    assert np.array_equal(out[4][0], out[8][0]) and np.array_equal(out[4][1], out[8][1])
    o.nprobe = 3
    _assert_same(*out[8], *o.search(xq, 20), "rows_inflight 8")


@pytest.mark.gpu
def test_sq8_factory_shards_through_the_client_with_embeddings():
    """IndexServer x2 on the GPU engine, faiss_factory "IVF{centroids},SQ8": return_embeddings
    carries the decoded winners, equal to the oracle's decode of the same shard"""
    import threading
    import time

    if EMU:
        pytest.skip("CUDA tensors")
    from distributed_faiss_b200.index_cfg import IndexCfg
    from distributed_faiss_b200.server import IndexServer
    from tests.test_gpu_api import free_ports, make_client, wait_listening, wait_trained
    import tempfile

    tmp = tempfile.TemporaryDirectory()
    ports = free_ports(2)
    servers = [IndexServer(r, tmp.name) for r in range(2)]
    for s, p in zip(servers, ports):
        threading.Thread(target=s.start_blocking, args=(p,), daemon=True).start()
    wait_listening(ports)
    try:
        rs = np.random.RandomState(16)
        d = 64
        client = make_client(ports)
        cfg = IndexCfg(faiss_factory="IVF{centroids},SQ8", dim=d, centroids=8, metric="l2", nprobe=4, train_num=400)
        client.create_index("sq8", cfg)
        for _ in range(2):
            x = clustered(rs, 600, d, ncl=8)
            client.add_index_data("sq8", x, list(range(600)), False)
        wait_trained(client, "sq8")
        t0 = time.time()
        while client.get_ntotal("sq8") != 1200:
            assert time.time() - t0 < 120, "adds never finished"
            time.sleep(0.05)
        wait_trained(client, "sq8")
        client.set_nprobe("sq8", 8)
        D, meta, embs = client.search(x[:5], 4, "sq8", return_embeddings=True)
        assert len(embs) == 5 and all(len(row) == 4 and all(e is not None for e in row) for row in embs)
        embs = np.asarray(embs, dtype=np.float32)
        decoded = set()
        for s in servers:
            ix = s.indexes["sq8"]
            o = S.make_index("ivf_sq8", d, metric=L2, nlist=8)
            o.set_state(ix.faiss_index.get_state())
            ids = np.arange(ix.faiss_index.ntotal, dtype=np.int64)
            rows = o.reconstruct_rows(ids)
            assert np.array_equal(ix.faiss_index.reconstruct_rows(ids), rows)
            decoded |= {r.tobytes() for r in rows}
        assert all(e.tobytes() in decoded for e in embs.reshape(-1, d))   # the winners' decoded rows
        client.close()
    finally:
        for s in servers:
            s.stop()
