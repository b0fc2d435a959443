"""fp16 scalar-quantized flat shards ("SQfp16", faiss IndexScalarQuantizer(d, QT_fp16, metric)).

The canonical answer of an SQfp16 shard is, bit for bit, the answer of a flat shard of the same metric
over the decoded rows x^ = fp16(x) (DESIGN.md section 2).  The CPU tests check the parser, the encoder,
the oracle, the host logic through oracle engines and the persistence; the `gpu` tests check the engine
against a DFX_FLAT shard built from the decoded rows, at every path (tensor-core screening FAST /
PRECISE / AUTO, the FFMA GEMM, range search, reconstruction)."""
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
from tests.oracle_flat_sq16 import OracleFlatSQ16, decode, encode, flat_sq16_engine_factory

IP, L2 = 0, 1
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMU = bool(os.environ.get("DFX_EMU_LIB"))


def _sz(full, emu):
    return emu if EMU else full


# ------------------------------------------------------------------ parser
@pytest.mark.parametrize("metric", [IP, L2])
def test_parser_maps_sqfp16_to_the_flat_sq16_kind(metric):
    assert "SQfp16" in ACCEPTED_FORMS
    assert parse_factory(64, "SQfp16", metric) == FactorySpec("flat_sq16", metric)
    spec = factory_spec(IndexCfg(faiss_factory="SQfp16", dim=32))               # the default metric is dot
    assert spec == FactorySpec("flat_sq16", IP)
    assert factory_spec(IndexCfg(faiss_factory="SQfp16", dim=32, metric="l2")) == FactorySpec("flat_sq16", L2)


@pytest.mark.parametrize("s", ["SQ8", "SQ4", "SQ6", "SQbf16", "SQfp16,RFlat", "SQfp16,Flat", "sqfp16", "SQfp16 "])
def test_other_scalar_quantizers_without_lists_stay_rejected(s):
    with pytest.raises(RuntimeError, match="accepted forms"):
        parse_factory(64, s, L2)


def test_ivf_gpu_refuses_sqfp16():
    with pytest.raises(RuntimeError, match="needs an IVF factory string"):
        factory_spec(IndexCfg(index_builder_type="ivf_gpu", faiss_factory="SQfp16", dim=32))


# ------------------------------------------------------------------ encoder
def _f16_reference(v):
    """round to nearest even into IEEE binary16, restated on float64 bit arithmetic (uint16 result)"""
    out = np.empty(v.shape, dtype=np.uint16)
    for i, x in enumerate(np.asarray(v, dtype=np.float64).reshape(-1)):
        sign = 0x8000 if np.signbit(x) else 0
        a = abs(x)
        if np.isnan(a):
            out.flat[i] = 0x7E00 | sign
            continue
        if a >= 65520.0:                                   # 65504 + half an ulp (2^4): rounds to inf
            out.flat[i] = 0x7C00 | sign
            continue
        e = max(int(np.floor(np.log2(a))) if a > 0 else -25, -14)   # subnormals share exponent -14
        ulp = 2.0 ** (e - 10)
        q = a / ulp
        r = np.floor(q)
        if q - r > 0.5 or (q - r == 0.5 and int(r) % 2 == 1):
            r += 1
        m = int(r)
        if m >= 2048:                                      # rounded up into the next binade
            m //= 2
            e += 1
        if m < 1024:                                       # subnormal (e == -14)
            bits = m
        else:
            bits = ((e + 15) << 10) | (m - 1024)
        out.flat[i] = bits | sign
    return out


def _special_values():
    tiny = np.float32(2.0 ** -24)
    vals = [0.0, -0.0, 1.0, -1.0, 65504.0, -65504.0, 65519.0, 65520.0, -65520.0, 1e9, -1e9, np.inf, -np.inf,
            tiny, -tiny, tiny * 0.5, tiny * 0.50001, tiny * 1.5, tiny * 2.5, 2.0 ** -14, 2.0 ** -14 * 0.999,
            1.0 + 2.0 ** -11, 1.0 + 3 * 2.0 ** -11, 1.0 + 2.0 ** -11 + 2.0 ** -20, 2049.0, 2051.0, 3.0e-8, 1e-10]
    rs = np.random.RandomState(5)
    return np.concatenate([np.array(vals, dtype=np.float32),
                           (rs.randn(2000) * 10.0 ** rs.uniform(-9, 5, 2000)).astype(np.float32)])


def test_numpy_float16_is_round_to_nearest_even_with_overflow_to_inf():
    v = _special_values()
    assert np.array_equal(encode(v), _f16_reference(v))
    assert np.isinf(decode(encode(v))[np.abs(v) >= 65520]).all()


# ------------------------------------------------------------------ oracle
@pytest.mark.parametrize("metric", [IP, L2])
def test_oracle_against_a_float64_restatement(metric, oracle_lib):
    rs = np.random.RandomState(3)
    d, n, k = 48, 700, 9
    xb, xq = rs.randn(n, d).astype(np.float32) * 3, rs.randn(13, d).astype(np.float32)
    o = OracleFlatSQ16(d, metric)
    o.add(xb[:300]); o.add(xb[300:])
    assert np.array_equal(o.codes16, encode(xb)) and o.ntotal == n
    D, I = o.search(xq, k)
    xh = decode(encode(xb)).astype(np.float64)
    ref = -(xq.astype(np.float64) @ xh.T) if metric == IP else ((xq[:, None, :].astype(np.float64) - xh[None]) ** 2).sum(-1)
    order = np.argsort(ref, axis=1, kind="stable")[:, :k]
    assert np.array_equal(I, order)
    want = np.take_along_axis(ref, order, 1)
    got = -D.astype(np.float64) if metric == IP else D.astype(np.float64)
    assert np.allclose(got, want, rtol=1e-4, atol=1e-3)
    assert np.array_equal(o.reconstruct_rows(I[0]), decode(encode(xb[I[0]])))


# ------------------------------------------------------------------ persistence
def _state(metric, n=57, d=24, seed=4):
    o = OracleFlatSQ16(d, metric)
    x = np.random.RandomState(seed).randn(n, d).astype(np.float32)
    x[3, 5] = 1e6                                                # an overflowed (inf) code
    o.add(x)
    return o, o.get_state()


@pytest.mark.parametrize("metric", [IP, L2])
def test_ixsq_byte_layout_round_trip(metric, tmp_path):
    o, st = _state(metric)
    assert st["kind"] == "flat_sq16" and st["metric"] == metric and st["codes16"].dtype == np.uint16
    path = str(tmp_path / "ix.faiss")
    faiss_io.write_index(st, path)
    raw = open(path, "rb").read()
    n, d = st["codes16"].shape
    want = b"IxSQ" + struct.pack("<iqqqBi", d, n, 1 << 20, 1 << 20, 1, metric) + struct.pack("<iif", 4, 0, 0.0)
    want += struct.pack("<QQ", d, 2 * d) + struct.pack("<Q", 0) + struct.pack("<Q", n * 2 * d)
    want += st["codes16"].astype("<u2").tobytes()
    assert raw == want
    back, nprobe = faiss_io.read_index(path)
    assert back["kind"] == "flat_sq16" and back["metric"] == metric and back["d"] == d
    assert np.array_equal(back["codes16"], st["codes16"])
    o2 = OracleFlatSQ16(d, metric)
    o2.set_state(back)
    q = np.random.RandomState(0).randn(5, d).astype(np.float32)
    assert all(a.tobytes() == b.tobytes() for a, b in zip(o.search(q, 6), o2.search(q, 6)))  # NaN too


def test_ixsq_refuses_other_quantizer_types(tmp_path):
    _, st = _state(L2, n=4, d=8)
    path = str(tmp_path / "ix.faiss")
    faiss_io.write_index(st, path)
    raw = bytearray(open(path, "rb").read())
    off = 4 + struct.calcsize("<iqqqBi")
    raw[off:off + 4] = struct.pack("<i", 0)                     # QT_8bit
    with pytest.raises(faiss_io.FaissFormatError, match="QT_fp16"):
        faiss_io.read_index(_write(tmp_path, raw))


def _write(tmp_path, raw):
    p = str(tmp_path / "bad.faiss")
    open(p, "wb").write(bytes(raw))
    return p


def _wait_added(ix):
    import time

    from distributed_faiss_b200.index_state import IndexState

    t0 = time.time()
    while ix.get_state() != IndexState.TRAINED:
        assert time.time() - t0 < 60
        time.sleep(0.02)


def _drop_stored_cfg(storage_dir):
    from distributed_faiss_b200.index import get_index_files

    os.remove(get_index_files(storage_dir)[3])


@pytest.mark.parametrize("fmt", ["dfx", "faiss"])
@pytest.mark.parametrize("metric", ["dot", "l2"])
def test_save_load_and_kind_mismatch_refusals(fmt, metric):
    rs = np.random.RandomState(6)
    d = 16
    with tempfile.TemporaryDirectory() as tmp:
        cfg = IndexCfg(faiss_factory="SQfp16", dim=d, metric=metric, index_storage_dir=tmp, index_format=fmt,
                       train_num=10)
        ix = Index(cfg, engine_factory=flat_sq16_engine_factory)
        x = rs.randn(300, d).astype(np.float32)
        ix.add_batch(x, list(range(300)), train_async_if_triggered=False)
        _wait_added(ix)
        assert isinstance(ix.faiss_index, OracleFlatSQ16) and ix.faiss_index.ntotal == 300
        D0, M0, _ = ix.search(x[:7], 5)
        ix.save()
        back = Index.from_storage_dir(tmp, cfg, engine_factory=flat_sq16_engine_factory)
        assert isinstance(back.faiss_index, OracleFlatSQ16)
        assert np.array_equal(back.faiss_index.codes16, encode(x))
        D1, M1, _ = back.search(x[:7], 5)
        assert np.array_equal(D0, D1) and M0 == M1
        # an SQfp16 shard under a cfg that builds fp32 flat, and the reverse (without the stored cfg, which
        # would otherwise stand in for a cfg that names no builder)
        _drop_stored_cfg(tmp)
        flat_cfg = IndexCfg(faiss_factory="Flat", dim=d, metric=metric, index_storage_dir=tmp, index_format=fmt)
        with pytest.raises(RuntimeError, match="refusing to load it"):
            Index.from_storage_dir(tmp, flat_cfg, engine_factory=flat_sq16_engine_factory)
    with tempfile.TemporaryDirectory() as tmp:
        flat_cfg = IndexCfg(faiss_factory="Flat", dim=d, metric=metric, index_storage_dir=tmp, index_format=fmt,
                            train_num=10)
        ix = Index(flat_cfg, engine_factory=flat_sq16_engine_factory)
        ix.add_batch(rs.randn(50, d).astype(np.float32), list(range(50)), train_async_if_triggered=False)
        _wait_added(ix)
        ix.save()
        _drop_stored_cfg(tmp)
        sq_cfg = IndexCfg(faiss_factory="SQfp16", dim=d, metric=metric, index_storage_dir=tmp, index_format=fmt)
        with pytest.raises(RuntimeError, match="refusing to load it"):
            Index.from_storage_dir(tmp, sq_cfg, engine_factory=flat_sq16_engine_factory)


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
        s = IndexServer(i, store.name, engine_factory=flat_sq16_engine_factory)
        threading.Thread(target=s.start_blocking, args=(p,), daemon=True).start()
        srv.append(s)
    wait_listening(ports)
    yield ports, srv
    for s in srv:
        s.stop()


@pytest.mark.parametrize("metric", ["dot", "l2"])
def test_sharded_search_through_servers_with_oracle_engines(servers, metric):
    """two shards behind IndexServers: the client's merged D and metadata equal the merge of the shards'
    own answers (the client negates for dot, as for every kind), with and without return_embeddings"""
    from oracle import oracle as O
    from tests.test_host_logic import make_client, wait_trained

    ports, srv = servers
    rs = np.random.RandomState(7)
    d, index_id = 32, f"sq16_{metric}"
    client = make_client(ports)
    client.create_index(index_id, IndexCfg(faiss_factory="SQfp16", dim=d, metric=metric, train_num=50))
    for b in range(4):
        client.add_index_data(index_id, clustered(rs, 200, d, ncl=8), [(b, i) for i in range(200)], False)
    client.sync_train(index_id)
    wait_trained(client, index_id)
    shards = [s.indexes[index_id] for s in srv]
    assert all(isinstance(ix.faiss_index, OracleFlatSQ16) and ix.faiss_index.metric == (IP if metric == "dot" else L2)
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
    "tests/test_flat_sq16.py::test_encode_matches_numpy_on_the_device",
    "tests/test_flat_sq16.py::test_bit_parity_with_a_flat_shard_of_the_decoded_rows[64-1024-0]",
    "tests/test_flat_sq16.py::test_bit_parity_with_a_flat_shard_of_the_decoded_rows[128-1024-1]",
    "tests/test_flat_sq16.py::test_near_duplicates_overflow_and_are_redone_exactly",
    "tests/test_flat_sq16.py::test_adds_between_searches_and_an_overflowed_code",
    "tests/test_flat_sq16.py::test_range_search_and_reconstruct_match_the_flat_shard",
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
                         cwd=ROOT, env=env, capture_output=True, text=True, timeout=1500)
    tail = (run.stdout + run.stderr)[-3000:]
    assert run.returncode == 0, tail
    assert f"{len(EMU_SUBSET)} passed" in run.stdout, tail


# ------------------------------------------------------------------ GPU: the engine
def _engine():
    from distributed_faiss_b200 import engine

    return engine


def _pair(d, metric, x):
    """(FLAT_SQ16 shard of x, DFX_FLAT shard of the decoded rows)"""
    E = _engine()
    g = E.GpuIndex(E.KIND_FLAT_SQ16, d, metric)
    f = E.GpuIndex(E.KIND_FLAT, d, metric)
    g.add(x)
    f.add(decode(encode(x)))
    return g, f


def _same(a, b, what):
    (Da, Ia), (Db, Ib) = a, b
    if not (np.array_equal(Ia, Ib) and np.array_equal(Da.view(np.uint32), Db.view(np.uint32))):
        bad = np.argwhere((Ia != Ib) | (Da.view(np.uint32) != Db.view(np.uint32)))
        q, j = bad[0]
        raise AssertionError(f"{what}: {len(bad)} slots differ; first q={q} j={j}: ({Da[q, j]!r},{Ia[q, j]}) vs "
                             f"({Db[q, j]!r},{Ib[q, j]})")


def _data(rs, n, d):
    x = clustered(rs, n, d, ncl=max(8, n // 400)) * np.float32(3)
    m = n // 20
    x[n - m:] = x[:m] + np.float32(1e-4) * rs.randn(m, d).astype(np.float32)   # near-duplicates
    return x


@pytest.mark.gpu
def test_encode_matches_numpy_on_the_device():
    """__float2half_rn on the device = np.float16: subnormals, ties to even, +-inf beyond 65504"""
    E = _engine()
    v = _special_values()
    v = np.resize(v, (len(v) + 63) // 64 * 64).reshape(-1, 64)
    g = E.GpuIndex(E.KIND_FLAT_SQ16, 64, L2)
    g.add(v)
    assert np.array_equal(g.get_array("codes16").reshape(v.shape), encode(v))
    assert g.get_state()["kind"] == "flat_sq16" and g.ntotal == v.shape[0]
    with pytest.raises(RuntimeError, match="must be 0"):
        E.GpuIndex(E.KIND_FLAT_SQ16, 64, L2, nlist=4)
    with pytest.raises(RuntimeError, match="must be 0"):
        E.GpuIndex(E.KIND_FLAT_SQ16, 64, L2, pq_nbits=8)


SHAPES = [(64, 1000), (64, 1024), (128, 1024), (128, 50_000), (128, 200_000), (768, 50_000), (2048, 1024),
          (2048, 50_000), (100, 1024), (100, 50_000)]


@pytest.mark.gpu
@pytest.mark.parametrize("metric", [IP, L2])
@pytest.mark.parametrize("d,n", SHAPES, ids=[f"{d}-{n}" for d, n in SHAPES])
def test_bit_parity_with_a_flat_shard_of_the_decoded_rows(metric, d, n):
    """every k, nq and screening mode: the SQfp16 shard returns the bits of the fp32 flat shard over x^"""
    rs = np.random.RandomState(d + n + metric)
    x = _data(rs, n, d)
    g, f = _pair(d, metric, x)
    xq = np.concatenate([x[:: max(1, n // 700)][:700], clustered(rs, 400, d, ncl=8)])[:1025]
    ks = (1, 10, 100, 101, 4096) if not EMU else (1, 10, 101)
    nqs = (1, 37, 1025) if not EMU else (1, 37)
    for nq in nqs:
        q = xq[:nq]
        for k in ks:
            want = f.search(q, k)
            for mode in (0, 1, 2):
                g.set_param("flat_tensor_cores", 1)
                g.set_param("tc_screen_mode", mode)
                _same(g.search(q, k), want, f"d={d} n={n} nq={nq} k={k} mode={mode}")
            g.set_param("flat_tensor_cores", 0)
            _same(g.search(q, k), want, f"d={d} n={n} nq={nq} k={k} FFMA")
    g.set_param("flat_tensor_cores", 1)


@pytest.mark.gpu
def test_near_duplicates_overflow_and_are_redone_exactly():
    E = _engine()
    rs = np.random.RandomState(9)
    d, n = 128, _sz(20_000, 2048)
    base = rs.randn(64, d).astype(np.float32)
    x = base[rs.randint(0, 64, n)] + np.float32(1e-3) * rs.randn(n, d).astype(np.float32)   # 64 tight clumps
    for metric in (IP, L2):
        g, f = _pair(d, metric, x)
        q = x[:50] + np.float32(1e-3)
        for mode in (2, 1, 0):
            g.set_param("tc_screen_mode", mode)
            _same(g.search(q, 10), f.search(q, 10), f"metric={metric} mode={mode}")
        # AUTO (mode 0, PRECISE on a new table) posts the statistics of its launches
        assert g.get_param("tc_stat_rows") == len(q) and g.get_param("tc_stat_overflow") > 0


@pytest.mark.gpu
def test_adds_between_searches_and_an_overflowed_code():
    E = _engine()
    rs = np.random.RandomState(10)
    d = 128
    for metric in (IP, L2):
        g = E.GpuIndex(E.KIND_FLAT_SQ16, d, metric)
        f = E.GpuIndex(E.KIND_FLAT, d, metric)
        q = rs.randn(20, d).astype(np.float32)
        for b in range(3):                                      # the screening table follows the adds
            x = rs.randn(int(rs.randint(700, 1500)), d).astype(np.float32)
            g.add(x)
            f.add(decode(encode(x)))
            for k in (1, 10):
                _same(g.search(q, k), f.search(q, k), f"metric={metric} batch={b} k={k}")
        # one input beyond 65504 encodes to inf: the shard answers what the FFMA GEMM answers
        x = rs.randn(5, d).astype(np.float32)
        x[2, 7] = 1e5
        g.add(x)
        f.add(decode(encode(x)))
        assert np.isinf(g.reconstruct_rows(np.array([g.ntotal - 3]))[0, 7])
        f.set_param("flat_tensor_cores", 0)
        for k in (1, 10):
            _same(g.search(q, k), f.search(q, k), f"metric={metric} inf code k={k}")


@pytest.mark.gpu
def test_oracle_parity():
    from oracle import oracle as O  # noqa: F401  (builds the oracle library)

    rs = np.random.RandomState(12)
    d, n = 128, _sz(30_000, 2048)
    x = _data(rs, n, d)
    for metric in (IP, L2):
        g, _ = _pair(d, metric, x)
        o = OracleFlatSQ16(d, metric)
        o.add(x)
        q = x[:33] + np.float32(0.01)
        for k in (1, 10, 100):
            _same(g.search(q, k), o.search(q, k), f"oracle metric={metric} k={k}")


@pytest.mark.gpu
def test_range_search_and_reconstruct_match_the_flat_shard():
    rs = np.random.RandomState(13)
    d, n = 128, _sz(40_000, 2048)
    x = _data(rs, n, d)
    for metric in (IP, L2):
        g, f = _pair(d, metric, x)
        q = x[:17] + np.float32(0.01)
        D, _ = f.search(q, 20)
        radius = float(np.median(D[:, -1]))
        for a, b in zip(g.range_search(q, radius), f.range_search(q, radius)):
            assert np.array_equal(a, b)
        Dg, Ig, R = g.search_and_reconstruct(q, 10)
        _same((Dg, Ig), f.search(q, 10), f"search_and_reconstruct metric={metric}")
        assert np.array_equal(R, decode(encode(x))[Ig])


@pytest.mark.gpu
def test_index_bytes_is_two_bytes_per_component():
    """N 2 d bytes of codes (+ 4 N of norms under L2) + the screening table's 4 d + 8 bytes (its zero mean
    and norm maximum), against the fp32 flat shard's 4 d of rows + 4 d of screening planes per vector"""
    E = _engine()
    rs = np.random.RandomState(14)
    d, n = 128, 4096
    x = rs.randn(n, d).astype(np.float32)
    for metric in (IP, L2):
        g, f = _pair(d, metric, x)
        norms = 4 * n if metric == L2 else 0
        assert g.get_param("index_bytes") == 2 * d * n + norms
        g.search(x[:3], 10)
        f.search(x[:3], 10)
        assert g.get_param("index_bytes") == 2 * d * n + norms + 4 * d + 8
        flat = f.get_param("index_bytes")
        print(f"metric={metric}: SQfp16 {g.get_param('index_bytes') / n:.1f} B/vector, fp32 flat {flat / n:.1f} B/vector")
        assert flat >= 8 * d * n


@pytest.mark.gpu
def test_client_over_sockets_and_the_search_plane():
    from distributed_faiss_b200.index_cfg import IndexCfg as Cfg
    from oracle import oracle as O
    from tests.test_gpu_api import _both_ways, _plane_cluster, wait_trained

    store, servers, plane, client = _plane_cluster(2)
    rs = np.random.RandomState(15)
    d = 128
    try:
        client.create_index("sq16", Cfg(faiss_factory="SQfp16", dim=d, train_num=10))   # the default metric, dot
        for b in range(4):
            client.add_index_data("sq16", clustered(rs, 1500, d, ncl=16), [(b, i) for i in range(1500)], False)
        client.sync_train("sq16")
        wait_trained(client, "sq16")
        shards = [s.indexes["sq16"] for s in servers]
        assert all(ix.faiss_index.kind == _engine().KIND_FLAT_SQ16 for ix in shards)
        q = clustered(rs, 40, d, ncl=16)
        per = [ix.faiss_index.search(q, 10) for ix in shards]
        Dall = np.stack([D for D, _ in per])
        pos = np.arange(Dall.size, dtype=np.int64).reshape(Dall.shape)
        Dref, P = O.merge(-Dall, pos)
        meta = [ix.id_to_metadata[i] if i >= 0 else None for ix, (_, I) in zip(shards, per) for i in I.reshape(-1)]
        rows = np.concatenate([ix.faiss_index.reconstruct_rows(I.reshape(-1)) for ix, (_, I) in zip(shards, per)])
        Mref = [[meta[p] if p >= 0 else None for p in row] for row in P]
        (Dp, Mp), (Ds, Ms) = _both_ways(client, plane, lambda: client.search(q, 10, "sq16"))
        for D, M in ((Dp, Mp), (Ds, Ms)):
            assert np.array_equal(D, Dref) and list(M) == Mref
        (Dp, Mp, Ep), (Ds, Ms, Es) = _both_ways(client, plane, lambda: client.search(q, 10, "sq16", True))
        for D, M, E in ((Dp, Mp, Ep), (Ds, Ms, Es)):
            assert np.array_equal(D, Dref) and list(M) == Mref
            assert np.array_equal(np.asarray(E).reshape(-1, d), rows[P.reshape(-1)])
    finally:
        client.close()
        plane.stop()
        for s in servers:
            s.stop()
