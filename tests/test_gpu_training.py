"""GPU training of every IVF kind, bit for bit against the restatement of the device build
(tests/oracle_train.py, DESIGN.md section 4.6a).

The search parity tests copy whatever the GPU trained into the oracle, so a wrong sample, seed,
residual or codebook would pass them.  Here the trained arrays themselves -- coarse centroids, PQ
codebooks, IVF-PQR refinement codebooks, the SQ8 range -- are compared byte for byte with what the
rules of the device build give on the same rows.

CPU: the restatement's random generator, sample and centroid update; the `gpu` tests run against
the emulated library.  GPU: the CUDA build against the restatement, including the tensor-core
assignment inside k-means and clusters of ~10^5 rows."""
import os
import platform
import shutil
import subprocess
import sys

import numpy as np
import pytest

from tests.conftest import clustered
from tests import oracle_train as T

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
IP, L2 = 0, 1
F32 = np.float32
EMU = bool(os.environ.get("DFX_EMU_LIB"))


def _sz(full, emu):
    return emu if EMU else full


# ------------------------------------------------------------------ the restatement, CPU
def test_mt19937_64_known_answer():
    rng = T.MT19937_64(5489)  # C++ [rand.predef]: the 10000th output of a default-constructed engine
    for _ in range(9999):
        rng()
    assert rng() == 9981545732273789042
    assert T.MT19937_64(0)() == 2947667278772165694


@pytest.mark.parametrize("n,k", [(1, 1), (10, 10), (1000, 37), (5000, 4096)])
def test_sample_rows_are_distinct_and_in_range(n, k):
    s = T.sample_rows(n, k, 1234)
    assert s.shape == (k,) and s.dtype == np.int64
    assert len(np.unique(s)) == k and s.min() >= 0 and s.max() < n
    assert not np.array_equal(s, T.sample_rows(n, k, 1235)) or k == n == 1
    assert np.array_equal(s[: k // 2], T.sample_rows(n, k // 2, 1234))  # a prefix of the same shuffle


def _f64_bound_check(cent, x, assign, skip=()):
    """|c - sum x / n_c| <= (n_c + 2) 2^-24 sum |x| / n_c per component, the fp32 sequential sum
    and the product with a rounded 1/n_c.  Returns (worst |c - mean| / bound, worst relative error)."""
    worst_ratio, worst_rel = 0.0, 0.0
    for c in range(cent.shape[0]):
        rows = x[assign == c].astype(np.float64)
        if len(rows) == 0 or c in skip:
            continue
        nc = len(rows)
        mean = rows.sum(0) / nc
        bound = (nc + 2) * 2.0 ** -24 * np.abs(rows).sum(0) / nc
        err = np.abs(cent[c].astype(np.float64) - mean)
        assert (err <= bound).all(), (c, nc, err.max(), bound[err.argmax()])
        worst_ratio = max(worst_ratio, float((err / np.maximum(bound, 1e-300)).max()))
        worst_rel = max(worst_rel, float((err / np.maximum(np.abs(mean), 1e-300)).max()))
    return worst_ratio, worst_rel


def test_restated_centroid_update_is_within_the_float64_bound():
    rs = np.random.RandomState(0)
    d, k = 12, 6
    sizes = [1, 2, 3, 700, 20000, 0]   # a single row, small clusters, a large one, an empty one
    x = np.concatenate([(rs.randn(s, d) * 10.0 ** rs.randint(-2, 3) + 100.0 * rs.randn(d)).astype(F32)
                        for s in sizes])
    a = np.repeat(np.arange(k), sizes)
    perm = rs.permutation(len(x))
    x, a = x[perm], a[perm]
    cent0 = rs.randn(k, d).astype(F32)
    cent, cnt = T.centroid_update(x, a, cent0)
    assert cnt.tolist() == sizes
    assert np.array_equal(cent[5], cent0[5])             # no rows: the centroid keeps its value
    assert np.array_equal(cent[0], x[a == 0][0])          # one row: that row
    _f64_bound_check(cent, x, a)
    # the sum is the sequential fp32 one: it is not the (more accurate) float64 sum rounded once
    big = x[a == 4].astype(np.float64)
    assert not np.array_equal(cent[4], (big.sum(0) / len(big)).astype(F32))


def test_restated_split_moves_the_big_cluster_by_one_1024th():
    cent = np.array([[1.0, 2.0, -4.0], [0, 0, 0], [8.0, 8.0, 8.0], [0, 0, 0]], dtype=F32)
    h = np.array([5, 0, 2, 0])
    splits = T.split_empty(cent, h)
    assert splits == [(1, 0), (3, 0)] and h.tolist() == [2, 2, 2, 1]   # ties of argmax -> the first
    e = 1 / 1024
    assert cent[3].tolist() == [(1 - e) * (1 + e), 2 * (1 + e) * (1 - e), -4 * (1 - e) * (1 + e)]
    assert cent[1].tolist() == [1 + e, 2 * (1 - e), -4 * (1 + e)]


# ------------------------------------------------------------------ GPU against the restatement
KINDS = {"ivf_flat": "KIND_IVF_FLAT", "ivf_sq": "KIND_IVF_SQ16", "ivf_sq8": "KIND_IVF_SQ8", "ivf_pq": "KIND_IVF_PQ",
         "ivf_pq_fs": "KIND_IVF_PQ_FS", "ivf_pqr": "KIND_IVF_PQR"}


def _gpu(kind, d, nlist, metric=L2, M=0, nbits=8, M2=0, rflat=False, **params):
    from distributed_faiss_b200 import engine as E

    g = E.GpuIndex(getattr(E, KINDS[kind]), d, metric, nlist=nlist, pq_m=M, pq_nbits=nbits, refine_m=M2,
                   refine_flat=rflat)
    for name, v in params.items():
        g.set_param(name, v)
    return g


def _trained(g, kind, d, M=0, nbits=8, M2=0):
    out = {"centroids": g.get_array("centroids").reshape(-1, d)}
    if kind in ("ivf_pq", "ivf_pq_fs", "ivf_pqr"):
        out["codebooks"] = g.get_array("codebooks").reshape(M, 1 << nbits, d // M)
    if kind == "ivf_pqr":
        out["refine_codebooks"] = g.get_array("refine_codebooks").reshape(M2, 256, d // M2)
    if kind == "ivf_sq8":
        out["sq_trained"] = g.get_array("sq_trained").reshape(2, d)
    return out


def _assert_same(got, want, what):
    assert sorted(got) == sorted(want), (what, sorted(got), sorted(want))
    for name in want:
        a, b = np.asarray(got[name], dtype=F32), np.asarray(want[name], dtype=F32)
        assert a.shape == b.shape, f"{what}: {name} has shape {a.shape}, the restatement {b.shape}"
        bad = np.argwhere(a.view(np.uint32) != b.view(np.uint32))
        if len(bad):
            i = tuple(int(v) for v in bad[0])
            raise AssertionError(f"{what}: {name} differs in {len(bad)} of {a.size} values; first at {i}: "
                                 f"gpu={float(a[i])!r} restatement={float(b[i])!r}")


def _train_both(kind, x, nlist, metric=L2, M=0, nbits=8, M2=0, niter=2, mpc=256, seed=None, log=None, **params):
    d = x.shape[1]
    if mpc != 256:
        params["max_points_per_centroid"] = mpc
    if seed is not None:
        params["train_seed"] = seed
    g = _gpu(kind, d, nlist, metric, M, nbits, M2, kmeans_niter=niter, **params)
    g.train(x)
    got = _trained(g, kind, d, M, nbits, M2)
    want = T.train(kind, x, nlist, metric, M, nbits, M2, niter, mpc, 1234 if seed is None else seed, log)
    return got, want


# kind, d, nlist, metric, M, nbits, M2, n (H100), n (emulator)
CASES = {
    "flat-l2": ("ivf_flat", 32, 16, L2, 0, 8, 0, 3000, 600),
    "flat-ip": ("ivf_flat", 32, 16, IP, 0, 8, 0, 3000, 600),
    "sq16-768": ("ivf_sq", 768, 8, L2, 0, 8, 0, 2000, 200),
    "sq8-l2": ("ivf_sq8", 64, 16, L2, 0, 8, 0, 3000, 600),
    "sq8-ip": ("ivf_sq8", 64, 16, IP, 0, 8, 0, 3000, 600),
    "pq8-64x16": ("ivf_pq", 64, 16, L2, 16, 8, 0, 3000, 600),       # dsub 4: DS = 4
    "pq8-48x16": ("ivf_pq", 48, 16, L2, 16, 8, 0, 3000, 600),       # dsub 3: the generic DS = 0
    "pq8-128x32-ip": ("ivf_pq", 128, 16, IP, 32, 8, 0, 3000, 600),  # residuals under the IP quantizer
    "pq8-768x128": ("ivf_pq", 768, 8, L2, 128, 8, 0, 2000, 300),    # wide, dsub 6
    "pq4-128x32": ("ivf_pq", 128, 16, L2, 32, 4, 0, 3000, 600),
    "fastscan-64x16": ("ivf_pq_fs", 64, 16, L2, 16, 4, 0, 3000, 600),
    "pqr-64-16+8": ("ivf_pqr", 64, 16, L2, 16, 8, 8, 3000, 600),
}


@pytest.mark.gpu
@pytest.mark.parametrize("case", list(CASES))
def test_training_matches_restatement(case):
    kind, d, nlist, metric, M, nbits, M2, n, n_emu = CASES[case]
    rs = np.random.RandomState(20)
    x = clustered(rs, _sz(n, n_emu), d, ncl=2 * nlist)
    got, want = _train_both(kind, x, nlist, metric, M, nbits, M2)
    _assert_same(got, want, case)


@pytest.mark.gpu
def test_rflat_trains_as_its_base_kind():
    rs = np.random.RandomState(21)
    d, nlist, M = 64, 16, 16
    x = clustered(rs, _sz(3000, 600), d, ncl=32)
    base = _gpu("ivf_pq", d, nlist, L2, M, kmeans_niter=2)
    rf = _gpu("ivf_pq", d, nlist, L2, M, rflat=True, kmeans_niter=2)
    base.train(x)
    rf.train(x)
    got = _trained(rf, "ivf_pq", d, M)
    _assert_same(got, _trained(base, "ivf_pq", d, M), "IVF-PQ,RFlat against IVF-PQ")
    _assert_same(got, T.train("ivf_pq", x, nlist, L2, M, 8, 0, 2), "IVF-PQ,RFlat")


@pytest.mark.gpu
@pytest.mark.parametrize("kind,M", [("ivf_flat", 0), ("ivf_pq", 8), ("ivf_sq8", 0)])
def test_training_on_a_subsample(kind, M):
    """n > max_points_per_centroid * nlist: k-means and the codec see a random subset of the rows"""
    rs = np.random.RandomState(22)
    d, nlist, mpc = 32, 16, 40
    x = clustered(rs, _sz(3000, 800), d, ncl=32)
    got, want = _train_both(kind, x, nlist, L2, M, mpc=mpc)
    _assert_same(got, want, f"{kind} sample of {mpc * nlist} rows")
    full = T.train(kind, x, nlist, L2, M, 8, 0, 2)  # without the sample: must differ, or the test is void
    assert not np.array_equal(full["centroids"], want["centroids"])


@pytest.mark.gpu
def test_pq_trains_on_a_prefix_of_the_sample():
    """4-bit PQ: 256 * 16 = 4096 rows train the codebooks, of nt > 4096 rows of the k-means sample"""
    rs = np.random.RandomState(23)
    d, nlist, M = 32, 32, 8
    x = clustered(rs, _sz(6000, 4500), d, ncl=64)
    got, want = _train_both("ivf_pq", x, nlist, L2, M, nbits=4)
    _assert_same(got, want, "pq4 on a prefix")


@pytest.mark.gpu
def test_training_follows_train_seed():
    rs = np.random.RandomState(24)
    d, nlist, M = 32, 16, 8
    x = clustered(rs, _sz(3000, 600), d, ncl=32)
    got, want = _train_both("ivf_pq", x, nlist, L2, M, seed=77)
    _assert_same(got, want, "train_seed 77")
    default, _ = _train_both("ivf_pq", x, nlist, L2, M)
    for name in ("centroids", "codebooks"):
        assert got[name].tobytes() != default[name].tobytes(), name


@pytest.mark.gpu
@pytest.mark.parametrize("niter", [1, 3])
def test_empty_clusters_are_split(niter):
    """40 distinct rows drawn over and over: the initial centroids repeat, the repeats get no rows
    (ties go to the smaller centroid) and are split off the largest cluster.  The `h[big] < 2` stop
    is out of reach here: with n >= k the halving keeps sum(h) = n, so some cluster always has >= 2."""
    rs = np.random.RandomState(25)
    d, nlist = 16, 64
    distinct = clustered(rs, 40, d, ncl=8)
    x = distinct[rs.randint(0, 40, size=_sz(2000, 600))]
    log = []
    got, want = _train_both("ivf_flat", x, nlist, niter=niter, log=log)
    assert log[0]["splits"], "the data must empty some clusters"
    _assert_same(got, want, f"splits, niter={niter}")
    if niter == 1:
        # the last split leaves its pair exactly +-1/1024 apart around the big cluster's centroid
        c, big = log[0]["splits"][-1]
        a, b = got["centroids"][c].astype(np.float64), got["centroids"][big].astype(np.float64)
        e = 1 / 1024
        up = np.where(np.arange(d) % 2 == 0, (1 + e) / (1 - e), (1 - e) / (1 + e))
        nz = b != 0
        assert nz.any() and np.allclose(a[nz] / b[nz], up[nz], rtol=1e-6, atol=0), (c, big, a / b)


@pytest.fixture(scope="module")
def tc_case():
    """nlist = 1024 at d = 64 sends k-means' assignment to the tensor cores; n is past one AUTO
    probe chunk of 16384 rows"""
    if EMU:
        pytest.skip("the emulator has no wgmma")
    rs = np.random.RandomState(26)
    x = clustered(rs, 20000, 64, ncl=512)
    return x, T.train("ivf_flat", x, 1024, L2, niter=2)


@pytest.mark.gpu
@pytest.mark.parametrize("tc,mode", [(1, 0), (1, 1), (1, 2), (0, 0)])
def test_tensor_core_assignment_inside_kmeans(tc_case, tc, mode):
    x, want = tc_case
    g = _gpu("ivf_flat", 64, 1024, kmeans_niter=2, tensor_cores=tc, tc_screen_mode=mode)
    g.train(x)
    _assert_same(_trained(g, "ivf_flat", 64), want, f"tensor_cores={tc} tc_screen_mode={mode}")


@pytest.mark.gpu
def test_large_clusters_are_exact_and_within_the_float64_bound():
    """4 clusters of ~50k rows each, offset by 100: the fp32 sums run long and large"""
    if EMU:
        pytest.skip("too large for the emulator")
    rs = np.random.RandomState(27)
    d, nlist, n = 16, 4, 200_000
    x = (clustered(rs, n, d, ncl=4) + F32(100)).astype(F32)
    log = []
    got, want = _train_both("ivf_flat", x, nlist, niter=2, mpc=100_000, log=log)
    last = log[-1]
    assert last["counts"].min() > 30_000 and not last["splits"]
    ratio, rel = _f64_bound_check(got["centroids"], x, last["assign"])
    _assert_same(got, want, f"large clusters (worst relative error to the float64 mean {rel:.3g}, "
                            f"{ratio:.3g} of the bound)")
    assert ratio <= 1.0, f"worst relative error {rel:.3g}"


@pytest.mark.gpu
def test_train_dev_and_repeated_training_give_the_same_bytes():
    if EMU:
        pytest.skip("CUDA tensors")
    import torch

    rs = np.random.RandomState(28)
    d, nlist, M, M2 = 64, 16, 16, 8
    x = clustered(rs, 3000, d, ncl=32)
    runs = []
    for dev in (False, False, True):
        g = _gpu("ivf_pqr", d, nlist, L2, M, 8, M2, kmeans_niter=2)
        if dev:
            g.train_dev(torch.from_numpy(x).cuda())
            torch.cuda.synchronize()
        else:
            g.train(x)
        runs.append(_trained(g, "ivf_pqr", d, M, 8, M2))
    _assert_same(runs[1], runs[0], "second training")
    _assert_same(runs[2], runs[0], "train_dev")
    _assert_same(runs[0], T.train("ivf_pqr", x, nlist, L2, M, 8, M2, 2), "ivf_pqr")


# ------------------------------------------------------------------ the gpu tests on the emulator
EMU_SUBSET = [
    "tests/test_gpu_training.py::test_training_matches_restatement[flat-l2]",
    "tests/test_gpu_training.py::test_training_matches_restatement[sq8-ip]",
    "tests/test_gpu_training.py::test_training_matches_restatement[pq8-64x16]",
    "tests/test_gpu_training.py::test_training_matches_restatement[pq8-48x16]",
    "tests/test_gpu_training.py::test_training_matches_restatement[pq4-128x32]",
    "tests/test_gpu_training.py::test_training_matches_restatement[fastscan-64x16]",
    "tests/test_gpu_training.py::test_training_matches_restatement[pqr-64-16+8]",
    "tests/test_gpu_training.py::test_training_on_a_subsample[ivf_flat-0]",
    "tests/test_gpu_training.py::test_empty_clusters_are_split[1]",
]


def test_training_gpu_tests_on_the_emulated_library():
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
