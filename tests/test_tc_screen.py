"""The coarse quantizer's tensor-core screening kernel (tc_coarse_kernel) against its own contract.

The exact decide stage after the screening hides most screening errors: a kernel that lost one
of PRECISE's three products would still give the oracle's probe lists on random data.  So the
summary is checked directly, through dfx_debug_tc_screen, against float64 ranking values
(L2: |c|^2 - 2 q.c, IP: -q.c) of every (query, group of 32 centroids):
  - gmin is within E of the group's exact minimum, gmin2 within E of its exact runner-up;
  - the column gargc names has an exact value within 2 E of the minimum;
  - gmin's 5 low bits are gargc, and columns past nlist never win.
E is the rigorous screening error of one ranking value: the bound screen_tol_rel (dfx_tc.cu)
is built from, without its 4 x 1.05 factor, plus the 2^-18 perturbation of the packed column
index and the rounding of the fp32 |c|^2 the kernel adds.
The emulated library serves the same entry point (emu_tc_screen), so the CPU suite runs the
`gpu` tests below against it as well (smaller batches).
"""
import ctypes as C
import os
import platform
import shutil
import subprocess
import sys

import numpy as np
import pytest

from tests.test_gpu_parity import EMU, _Dev

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
L2, IP = 1, 0
NLIST = 1100  # 1152 padded columns: group 34 is partly padding, group 35 entirely
BIG = 3.0e38  # the kernel's value of a padded column


def _screen_err_rel(d, npl):
    """screen_tol_rel's bound of |q.c - screen| / (|q| max|c|), before its 4.2 factor"""
    return (2.0 ** -10 + 2.0 ** -22 + d * 2.0 ** -24) if npl == 1 else (3 * 2.0 ** -22 + 3 * d * 2.0 ** -24)


def _index(d, metric, cent):
    from distributed_faiss_b200 import engine as E

    g = E.GpuIndex(E.KIND_IVF_FLAT, d, metric, nlist=cent.shape[0])
    g.set_state({"centroids": cent, "list_off": np.zeros(cent.shape[0] + 1, np.int64), "ids": np.zeros(0, np.int64),
                 "vecs": np.zeros((0, d), np.float32)})
    return g


def _screen(g, xq, npl):
    from distributed_faiss_b200 import engine as E

    nq, ng = xq.shape[0], -(-g.nlist // 128) * 4
    x = _Dev(xq)
    gmin, gmin2 = _Dev(np.zeros((nq, ng), np.float32)), _Dev(np.zeros((nq, ng), np.float32))
    gargc = _Dev(np.zeros((nq, ng), np.uint8))
    E._check(E.lib().dfx_debug_tc_screen(g._h, C.c_int64(nq), C.c_void_p(x.ptr), C.c_int(npl), C.c_void_p(gmin.ptr),
                                         C.c_void_p(gmin2.ptr), C.c_void_p(gargc.ptr)))
    return gmin.get(), gmin2.get(), gargc.get()


def _check_summary(xq, cent, metric, npl, gmin, gmin2, gargc, what):
    nq, d = xq.shape
    nlist, ng = cent.shape[0], gmin.shape[1]
    q, c = xq.astype(np.float64), cent.astype(np.float64)
    cn = (c * c).sum(1)
    V = (cn[None, :] - 2.0 * (q @ c.T)) if metric == L2 else -(q @ c.T)
    Vp = np.full((nq, ng * 32), np.inf)
    Vp[:, :nlist] = V
    G = Vp.reshape(nq, ng, 32)
    Gs = np.sort(G, axis=2)
    cmax2 = cn.max()
    s = np.sqrt((q * q).sum(1) * cmax2)[:, None]
    E = ((2.0 if metric == L2 else 1.0) * _screen_err_rel(d, npl) * s + 2.0 ** -18 * (cmax2 + 2.0 * s)
         + d * 2.0 ** -24 * cmax2)
    real = np.arange(ng) * 32 < nlist  # groups with at least one real column
    g1, g2 = gmin.astype(np.float64), gmin2.astype(np.float64)
    # the packing: gmin carries its own column in the 5 low bits
    assert np.array_equal(gmin.view(np.uint32) & 31, gargc.astype(np.uint32)), what
    bad = np.abs(g1 - Gs[:, :, 0])[:, real] > E
    assert not bad.any(), f"{what}: gmin off by more than the screening error at {np.argwhere(bad)[:5]}"
    both = np.isfinite(Gs[:, :, 1]) & real[None, :]
    bad2 = both & (np.abs(g2 - np.where(both, Gs[:, :, 1], 0.0)) > E)
    assert not bad2.any(), f"{what}: gmin2 off by more than the screening error at {np.argwhere(bad2)[:5]}"
    col = np.arange(ng)[None, :] * 32 + gargc.astype(np.int64)
    assert (col[:, real] < nlist).all(), f"{what}: a padded column won its group"
    picked = np.take_along_axis(Vp, np.minimum(col, nlist - 1), axis=1)
    bad3 = (picked - Gs[:, :, 0] > 2 * E) & real[None, :]
    assert not bad3.any(), f"{what}: gargc names a column far from the minimum at {np.argwhere(bad3)[:5]}"
    assert (g1[:, ~real] >= BIG * 0.99).all() and (g2[:, ~real] >= BIG * 0.99).all(), what


def _queries(rs, cent, nq, d):
    near = cent[rs.randint(0, cent.shape[0], nq)] + 0.05 * rs.randn(nq, d)
    far = 3.0 * rs.randn(nq, d)
    return np.where((np.arange(nq) % 4 == 3)[:, None], far, near).astype(np.float32)


NQS = (1, 37, 300) if EMU else (1, 37, 4096 + 37)


@pytest.mark.gpu
@pytest.mark.parametrize("d", [64, 128, 256])
@pytest.mark.parametrize("metric", [L2, IP])
@pytest.mark.parametrize("npl", [1, 2])
def test_screening_summary_is_within_the_error_bound(d, metric, npl):
    """every resident shape (and the streamed PRECISE d = 256), batches of 1, 37 and 4096 + 37
    queries (partial query tiles), nlist 1100 (partial and fully padded groups)"""
    rs = np.random.RandomState(1000 + d + 10 * metric + npl)
    cent = (rs.randn(NLIST, d) * (1.0 + rs.rand(NLIST, 1))).astype(np.float32)
    g = _index(d, metric, cent)
    for nq in NQS:
        xq = _queries(rs, cent, nq, d)
        _check_summary(xq, cent, metric, npl, *_screen(g, xq, npl), f"d={d} metric={metric} npl={npl} nq={nq}")


@pytest.mark.gpu
@pytest.mark.parametrize("npl", [1, 2])
def test_screening_summary_with_duplicate_centroids(npl):
    """exact ties inside and across groups: 40 copies of one centroid, some sharing a group"""
    rs = np.random.RandomState(7 + npl)
    d = 128
    cent = rs.randn(NLIST, d).astype(np.float32)
    cols = np.concatenate([np.arange(0, 1100, 29), [1, 2, 3]])
    cent[cols] = cent[5]
    g = _index(d, L2, cent)
    xq = np.concatenate([cent[5][None] + 0.01 * rs.randn(60, d), _queries(rs, cent, 70, d)]).astype(np.float32)
    _check_summary(xq, cent, L2, npl, *_screen(g, xq, npl), f"duplicates npl={npl}")


def test_screening_contract_on_the_emulated_library():
    """the tests above against emu_tc_screen, the CPU emulator's restatement of the kernel's result"""
    if EMU:
        pytest.skip("already running against the emulated library")
    if shutil.which("g++") is None or platform.machine() != "x86_64":
        pytest.skip("the emulator needs g++ on x86-64")
    sys.path.insert(0, os.path.join(ROOT, "tests", "emu"))
    try:
        import build_emu_lib
    finally:
        sys.path.pop(0)
    env = dict(os.environ, DFX_EMU_LIB=build_emu_lib.build(), DFX_EXPERIMENTAL="1")
    run = subprocess.run([sys.executable, "-m", "pytest", "-m", "gpu", "-q", "-p", "no:cacheprovider",
                          os.path.join("tests", "test_tc_screen.py")], cwd=ROOT, env=env, capture_output=True,
                         text=True, timeout=1500)
    tail = (run.stdout + run.stderr)[-3000:]
    assert run.returncode == 0, tail
    assert "14 passed" in run.stdout, tail
