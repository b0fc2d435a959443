"""The coarse quantizer's decide stage on the tensor-core search path (dfx_tc.cu,
decide_rows_kernel): the G smallest screening groups of a row, its threshold and overflow test, and
the exact re-rank of the surviving centroids, in one kernel.  The probe lists must be exactly the
oracle's coarse top-nprobe at FAST and PRECISE screening, for nprobe up to 32, through each source
of a row's groups:
  - selected in the kernel in two levels (G <= 32 of 128 or more groups of 32 centroids: nlist 4096
    and 65 536 up to nprobe 24);
  - selected in the kernel in one level (G <= 32 of 32 to 124 groups: nlist 1024, and nlist 3200
    up to nprobe 24);
  - given by the radix select (33 <= G <= 64: nlist 2048, where every one of the 64 groups is kept,
    and nprobe 32 at 3200 lists and more, G = 40).
Rows with more near-tied groups than kept ones must still be redone over all centroids, and the
AUTO precision's counters must count them.

Each list of the shard holds exactly one vector (its centroid), so a search with k = nprobe returns
the ids of the probed lists: the probe keys themselves, not only what the list scan makes of them.

The `gpu` tests also run on the CPU emulator (tests/emu/, the product sources compiled by g++):
test_decide_on_the_emulated_library runs them there in a subprocess.
"""
import os
import platform
import shutil
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMU = bool(os.environ.get("DFX_EMU_LIB"))
IP, L2 = 0, 1


def _shard(nlist, d, metric, ndup, seed):
    """(gpu index, oracle index, centroids): random centroids, `ndup` copies of centroid 0's value
    spread over `ndup` groups of 32 (at descending positions inside their groups, so that the
    packed column index orders the screening values against the id order), one vector per list"""
    from distributed_faiss_b200 import engine as E
    from oracle import oracle as O

    rs = np.random.RandomState(seed)
    cent = rs.randn(nlist, d).astype(np.float32)
    dup = 32 * np.arange(ndup) + (31 - np.arange(ndup) % 32)
    cent[dup] = cent[dup[0]]
    st = {"centroids": cent, "list_off": np.arange(nlist + 1, dtype=np.int64),
          "ids": np.arange(nlist, dtype=np.int64), "vecs": cent.copy()}
    g = E.GpuIndex(E.KIND_IVF_FLAT, d, metric, nlist=nlist)
    g.set_state(st)
    o = O.make_index("ivf_flat", d, metric=metric, nlist=nlist)
    o.set_state(st)
    return g, o, cent, dup


def _queries(rs, cent, dup, nclean, ndup_rows):
    """rows near random other centroids, then rows near the duplicated one (more near-ties than
    kept groups)"""
    d = cent.shape[1]
    others = np.setdiff1d(np.arange(cent.shape[0]), dup)
    clean = cent[others[rs.randint(0, others.size, nclean)]] + 0.1 * rs.randn(nclean, d)
    near = cent[dup[0]][None] + 0.01 * rs.randn(ndup_rows, d)
    return np.concatenate([clean, near]).astype(np.float32)


def _check(g, o, cent, xq, metric, nprobe, what):
    from oracle import oracle as O

    g.nprobe = nprobe
    o.nprobe = nprobe
    Dg, Ig = g.search(xq, nprobe)
    Do, Io = o.search(xq, nprobe)
    assert np.array_equal(Ig, Io) and np.array_equal(Dg, Do), what
    assert g.last_stats()["ndis"] == o.last_ndis == xq.shape[0] * nprobe, what
    keys, _ = O.coarse(metric, cent, xq, nprobe)  # the exact coarse top-nprobe
    assert np.array_equal(np.sort(Ig, axis=1), np.sort(keys, axis=1)), what


def _fast_tol(q, cent):
    """an upper bound of dfx_tc.cu's FAST tolerance of each row (screen_tol, L2, centred)"""
    d = cent.shape[1]
    m = cent.astype(np.float64).mean(0)
    cmax2 = float((cent.astype(np.float64) ** 2).sum(1).max())
    cmax2c = float(((cent - m) ** 2).sum(1).max())
    s = np.sqrt((q.astype(np.float64) ** 2).sum(1) * cmax2)
    sc = np.sqrt(((q - m) ** 2).sum(1) * cmax2c)
    err = 2.0 ** -10 + 2.0 ** -22 + d * 2.0 ** -24
    return (4.2 * (err + 2.0 ** -23) * sc + 2.1 * (2.0 ** -18 + 2.0 ** -23) * (cmax2c + 2 * sc)
            + 2.1 * (2.0 ** -17 + 2.0 ** -22 + d * 2.0 ** -24) * (cmax2 + 2 * s)) * 1.01


def _clear_of_overflow(q, cent, nprobe, G):
    """rows whose exact G-th smallest group minimum lies more than two FAST tolerances above the
    nprobe-th: no screening error can make them overflow (the tolerance is twice the error bound)"""
    v = (cent.astype(np.float64) ** 2).sum(1)[None] - 2.0 * q.astype(np.float64) @ cent.astype(np.float64).T
    gm = np.sort(v.reshape(q.shape[0], -1, 32).min(2), axis=1)
    return gm[:, G - 1] - gm[:, nprobe - 1] > 2.0 * _fast_tol(q, cent)


# 32, 64, 100, 128 and 2048 groups of 32 lists
CASES = [(1024, L2), (2048, IP), (3200, L2), (4096, L2), (4096, IP), (65536, L2)]


@pytest.mark.gpu
@pytest.mark.parametrize("nlist,metric", CASES)
def test_probe_keys_are_the_exact_coarse_top_nprobe(nlist, metric):
    d = 64
    g, o, cent, dup = _shard(nlist, d, metric, min(40, nlist // 32), seed=5)
    rs = np.random.RandomState(6)
    xq = _queries(rs, cent, dup, 24 if EMU else 500, 2 if (EMU and nlist > 4096) else 8)
    for nprobe in (1, 8, 16, 24, 32):
        for mode, name in ((2, "precise"), (1, "fast")):
            g.set_param("tc_screen_mode", mode)
            _check(g, o, cent, xq, metric, nprobe, f"nlist={nlist} metric={metric} nprobe={nprobe} {name}")


@pytest.mark.gpu
@pytest.mark.parametrize("nlist", [3200, 4096, 65536])
def test_overflow_rows_are_redone_and_counted_by_auto(nlist):
    """AUTO (tc_screen_mode 0) starts PRECISE and counts, per launch, the rows that overflow and
    those that FAST would overflow; clean rows move it to FAST once the window is full, a FAST launch
    that overflows moves it back.  The rows near the duplicated centroid overflow at either
    precision (48 exactly tied groups, 32 kept); the clean rows are the random rows clear of it
    (all but one of 1024 at 3200 lists, all at the other sizes)."""
    d, nprobe = 64, 8
    g, o, cent, dup = _shard(nlist, d, L2, 48, seed=7)
    rs = np.random.RandomState(8)
    nclean, nnear = (32, 2) if EMU else (1024, 24)
    xq = _queries(rs, cent, dup, nclean, nnear)
    G = min(32, nprobe + 24)
    keep = _clear_of_overflow(xq[:nclean], cent, nprobe, G)
    assert keep.sum() >= nclean - 1
    xq = np.concatenate([xq[:nclean][keep], xq[nclean:]])
    nclean = int(keep.sum())
    clean = xq[:nclean]
    g.set_param("tc_screen_mode", 0)
    g.set_param("tc_auto_window", 2 * nclean)
    assert g.get_param("tc_fast") == 0.0
    for it in range(2):                                        # clean rows fill the window: FAST
        _check(g, o, cent, clean, L2, nprobe, f"auto clean {it}")
        assert g.get_param("tc_stat_rows") == nclean
        assert g.get_param("tc_stat_overflow") == 0 and g.get_param("tc_stat_fast_would") == 0
    assert g.get_param("tc_fast") == 1.0
    _check(g, o, cent, xq, L2, nprobe, "auto at FAST with overflowing rows")
    assert g.get_param("tc_stat_rows") == nclean + nnear
    assert g.get_param("tc_stat_overflow") == nnear
    assert g.get_param("tc_fast") == 0.0                       # more than 1 in the window: back to PRECISE
    _check(g, o, cent, xq, L2, nprobe, "auto at PRECISE with overflowing rows")
    assert g.get_param("tc_stat_overflow") == nnear and g.get_param("tc_stat_fast_would") == nnear
    assert g.get_param("tc_fast") == 0.0


def test_decide_on_the_emulated_library():
    if shutil.which("g++") is None or platform.machine() != "x86_64":
        pytest.skip("the emulator needs g++ on x86-64")
    sys.path.insert(0, os.path.join(ROOT, "tests", "emu"))
    try:
        import build_emu_lib
    finally:
        sys.path.pop(0)
    env = dict(os.environ, DFX_EMU_LIB=build_emu_lib.build())
    run = subprocess.run([sys.executable, "-m", "pytest", "-m", "gpu", "-q", "-x", "-p", "no:cacheprovider",
                          os.path.join("tests", "test_tc_decide.py")],
                         cwd=ROOT, env=env, capture_output=True, text=True, timeout=1500)
    tail = (run.stdout + run.stderr)[-3000:]
    assert run.returncode == 0, tail
    assert "9 passed" in run.stdout, tail
