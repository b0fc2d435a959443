"""The coarse quantizer's screening centred on the mean m of its table (dfx_tc.cu).

Rows shaped like the bench's generator, mu + A z + noise with |mu|^2 much larger than the spread
|A z|^2, are where centring matters: the tensor cores see q - m and c - m, and the summary is
moved back to the original ranking frame by a per-row term.  Checked here:
  - probe lists and search results stay bit-identical to the oracle at FAST, PRECISE and AUTO;
  - the summary is within the centred error bound, which the raw screening misses on this data;
  - AUTO settles on FAST on such data;
  - duplicate centroids still go through the exact fallback;
  - rows added through the tensor-core assignment land in the oracle's lists.
The emulated library serves the same entry points, so the CPU suite runs the `gpu` tests below
against it as well (smaller sizes).
"""
import os
import platform
import shutil
import subprocess
import sys

import numpy as np
import pytest

from tests.test_gpu_parity import EMU, _assert_same, _engine
from tests.test_tc_screen import _index, _screen

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
L2 = 1
D, R = 128, 16


def _offset_rows(rs, n, mu, A, spread=1.0, noise=0.01):
    return (mu[None, :] + spread * rs.randn(n, R) @ A.T + noise * rs.randn(n, D)).astype(np.float32)


def _frame(rs, offset):
    A = np.linalg.qr(rs.randn(D, R))[0]
    return offset * rs.randn(D), A


def _ivf(cent, xb):
    from oracle import oracle as O

    E = _engine()
    nlist = cent.shape[0]
    empty = {"centroids": cent, "list_off": np.zeros(nlist + 1, np.int64), "ids": np.zeros(0, np.int64),
             "vecs": np.zeros((0, D), np.float32)}
    o = O.make_index("ivf_flat", D, metric=L2, nlist=nlist)
    o.set_state(empty)
    g = E.GpuIndex(E.KIND_IVF_FLAT, D, L2, nlist=nlist)
    g.set_state(empty)
    o.add(xb)
    g.add(xb)  # dfx_tc_assign
    return g, o


@pytest.mark.gpu
def test_offset_data_matches_oracle_in_every_mode():
    """bench-like rows (|mu|^2 ~ 128, spread ~ 16): lists built by the tensor-core assignment and
    search results at nprobe 1, 8 and 32 are the oracle's, FAST, PRECISE and AUTO alike"""
    rs = np.random.RandomState(5)
    mu, A = _frame(rs, 1.0)
    nlist = 4096
    cent = _offset_rows(rs, nlist, mu, A)
    xb = _offset_rows(rs, 3000 if EMU else 40_000, mu, A)
    g, o = _ivf(cent, xb)
    st = g.get_state()
    assert np.array_equal(st["list_off"], o.list_off) and np.array_equal(st["ids"], o.ids)
    xq = _offset_rows(rs, 40 if EMU else 500, mu, A)
    for nprobe in (1, 8, 32):
        g.nprobe = nprobe
        o.nprobe = nprobe
        Do, Io = o.search(xq, 10)
        for mode in (2, 1, 0):
            g.set_param("tc_screen_mode", mode)
            _assert_same(*g.search(xq, 10), Do, Io, f"offset data nprobe={nprobe} mode={mode}")
            assert g.last_stats()["ndis"] == o.last_ndis


@pytest.mark.gpu
@pytest.mark.parametrize("npl", [1, 2])
def test_summary_is_within_the_centred_bound(npl):
    """|mu|^2 ~ 8 000: the centred bound 2 (err + 2^-23) |q-m| max|c-m| plus 2^-17 of the magnitudes
    in both frames is about 0.2 at FAST, while the raw screening's fp16 rounding of q.c ~ 8 000
    misses the float64 values by more than that"""
    rs = np.random.RandomState(11 + npl)
    mu, A = _frame(rs, 8.0)
    nlist = 1100
    cent = _offset_rows(rs, nlist, mu, A)
    xq = _offset_rows(rs, 37 if EMU else 300, mu, A)
    g = _index(D, L2, cent)
    gmin, gmin2, gargc = _screen(g, xq, npl)
    q, c = xq.astype(np.float64), cent.astype(np.float64)
    m = c.mean(0)
    V = (c * c).sum(1)[None, :] - 2.0 * q @ c.T
    ng = gmin.shape[1]
    Vp = np.full((xq.shape[0], ng * 32), np.inf)
    Vp[:, :nlist] = V
    Gs = np.sort(Vp.reshape(xq.shape[0], ng, 32), axis=2)
    sc = np.sqrt(((q - m) ** 2).sum(1) * ((c - m) ** 2).sum(1).max())[:, None]
    vc = ((c - m) ** 2).sum(1).max() + 2.0 * sc
    rq = np.abs((m * m).sum() - 2.0 * q @ m)[:, None]
    err = (2.0 ** -10 + 2.0 ** -22 + D * 2.0 ** -24) if npl == 1 else (3 * 2.0 ** -22 + 3 * D * 2.0 ** -24)
    real = np.arange(ng) * 32 < nlist
    for got, want in ((gmin, Gs[:, :, 0]), (gmin2, Gs[:, :, 1])):
        E = 2.0 * (err + 2.0 ** -23) * sc + 2.0 ** -17 * (vc + np.abs(want) + rq)
        ok = np.isfinite(want) & real[None, :]
        bad = ok & (np.abs(got.astype(np.float64) - np.where(ok, want, 0.0)) > E)
        assert not bad.any(), f"npl={npl}: off by more than the centred bound at {np.argwhere(bad)[:5]}"
    assert np.array_equal(gmin.view(np.uint32) & 31, gargc.astype(np.uint32))


@pytest.mark.gpu
def test_auto_moves_to_fast_on_offset_data():
    """the bench's kind of data: with the screening centred, FAST's tolerance leaves no row with
    more near-ties than kept groups, so AUTO settles on FAST after a window of rows"""
    E = _engine()
    rs = np.random.RandomState(17)
    mu, A = _frame(rs, 1.0)
    nlist = 4096
    cent = _offset_rows(rs, nlist, mu, A)
    g = E.GpuIndex(E.KIND_IVF_FLAT, D, L2, nlist=nlist)
    g.set_state({"centroids": cent, "list_off": np.zeros(nlist + 1, np.int64), "ids": np.zeros(0, np.int64),
                 "vecs": np.zeros((0, D), np.float32)})
    g.nprobe = 8
    nb = 128 if EMU else 4096
    g.set_param("tc_auto_window", 3 * nb)
    would = 0.0
    for it in range(4):
        g.search(_offset_rows(rs, nb, mu, A), 10)
        would += g.get_param("tc_stat_fast_would")
    assert would == 0.0 and g.get_param("tc_fast") == 1.0


@pytest.mark.gpu
def test_duplicate_offset_centroids_take_the_exact_fallback():
    """40 copies of one centroid among offset rows: more near-ties than kept groups, so the rows
    near it are redone over all lists; results stay the oracle's in every mode"""
    rs = np.random.RandomState(19)
    mu, A = _frame(rs, 1.0)
    nlist = 4096
    cent = _offset_rows(rs, nlist, mu, A)
    cols = 32 * np.arange(40) + (31 - np.arange(40) % 32)
    cent[cols] = cent[cols[0]]
    xb = _offset_rows(rs, 2000 if EMU else 20_000, mu, A)
    xb[:100] = cent[cols[0]] + 0.01 * rs.randn(100, D).astype(np.float32)
    g, o = _ivf(cent, xb)
    st = g.get_state()
    assert np.array_equal(st["list_off"], o.list_off) and np.array_equal(st["ids"], o.ids)
    xq = np.concatenate([cent[cols[0]][None] + 0.001 * rs.randn(20, D), _offset_rows(rs, 20, mu, A)])
    xq = xq.astype(np.float32)
    for nprobe in (1, 8, 32):
        g.nprobe = nprobe
        o.nprobe = nprobe
        Do, Io = o.search(xq, 10)
        for mode in (2, 1, 0):
            g.set_param("tc_screen_mode", mode)
            _assert_same(*g.search(xq, 10), Do, Io, f"duplicates nprobe={nprobe} mode={mode}")


def test_centring_on_the_emulated_library():
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
                          os.path.join("tests", "test_tc_center.py")], cwd=ROOT, env=env, capture_output=True,
                         text=True, timeout=1500)
    tail = (run.stdout + run.stderr)[-3000:]
    assert run.returncode == 0, tail
    assert "5 passed" in run.stdout, tail
