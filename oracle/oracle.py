"""CPU ORACLE bindings (test infrastructure -- NOT product code).

ctypes wrapper over oracle/libdfx_oracle.so (built from oracle/dfx_oracle.c by
oracle/Makefile) plus small faiss-shaped index classes so that the tests can
drive "the reference's CPU path" through the same surface that
distributed_faiss/index.py uses on a faiss object
(`.train/.add/.search/.ntotal/.nprobe/.nlist/.quantizer.reconstruct_n`,
reference index.py:184,217,255-257,350,356,425).

Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline /
`--impl reference` legs may import this module.  PARITY STATUS: see the
header of dfx_oracle.c (merge pinned by the reference's golden vectors; the
IVF arithmetic is "parity unpinned" against real faiss).
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

from distributed_faiss_b200.engine import STATE_ARRAYS, StateLayout

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB_PATH = os.path.join(_HERE, "libdfx_oracle.so")

METRIC_IP = 0
METRIC_L2 = 1
FLT_MAX = float(np.finfo(np.float32).max)


def build(force: bool = False) -> str:
    src = os.path.join(_HERE, "dfx_oracle.c")
    if force or (not os.path.exists(_LIB_PATH)) or os.path.getmtime(_LIB_PATH) < os.path.getmtime(src):
        subprocess.check_call(["make", "-C", _HERE, "-B"], stdout=subprocess.DEVNULL)
    return _LIB_PATH


_lib = None


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(_LIB_PATH):
            build()
        _lib = C.CDLL(_LIB_PATH)
        _lib.orc_warp_dot.restype = C.c_float
        _lib.orc_warp_dot_h.restype = C.c_float
    return _lib


def _p(a):
    return a.ctypes.data_as(C.c_void_p) if a is not None else None


def _f32(x):
    return np.ascontiguousarray(x, dtype=np.float32)


def _i64(x):
    return np.ascontiguousarray(x, dtype=np.int64)


def num_threads() -> int:
    return int(lib().orc_num_threads())


# ---------------------------------------------------------------- primitives
def warp_dot(a, b, mode):
    a, b = _f32(a), _f32(b)
    return float(lib().orc_warp_dot(_p(a), _p(b), C.c_int(a.shape[0]), C.c_int(mode)))


def float_to_half(x):
    x = _f32(x)
    out = np.empty(x.shape, dtype=np.uint16)
    lib().orc_float_to_half(_p(x), _p(out), C.c_int64(x.size))
    return out


def half_to_float(h):
    h = np.ascontiguousarray(h, dtype=np.uint16)
    out = np.empty(h.shape, dtype=np.float32)
    lib().orc_half_to_float(_p(h), _p(out), C.c_int64(h.size))
    return out


def flat_search(metric, xb, xq, k):
    xb, xq = _f32(xb), _f32(xq)
    nq, d = xq.shape
    D = np.empty((nq, k), dtype=np.float32)
    I = np.empty((nq, k), dtype=np.int64)
    lib().orc_flat_search(C.c_int(metric), C.c_int(d), C.c_int64(xb.shape[0]), _p(xb), C.c_int64(nq),
                          _p(xq), C.c_int64(k), _p(D), _p(I))
    return D, I


def coarse(metric, cent, xq, nprobe):
    cent, xq = _f32(cent), _f32(xq)
    nq, d = xq.shape
    keys = np.empty((nq, nprobe), dtype=np.int64)
    vals = np.empty((nq, nprobe), dtype=np.float32)
    lib().orc_coarse(C.c_int(metric), C.c_int(d), C.c_int64(cent.shape[0]), _p(cent), C.c_int64(nq),
                     _p(xq), C.c_int64(nprobe), _p(keys), _p(vals))
    return keys, vals


def assign(metric, cent, x):
    cent, x = _f32(cent), _f32(x)
    out = np.empty((x.shape[0],), dtype=np.int64)
    lib().orc_assign(C.c_int(metric), C.c_int(x.shape[1]), C.c_int64(cent.shape[0]), _p(cent),
                     C.c_int64(x.shape[0]), _p(x), _p(out))
    return out


def kmeans(x, k, niter=25, seed=1234):
    x = _f32(x)
    n, d = x.shape
    cent = np.empty((k, d), dtype=np.float32)
    rc = lib().orc_kmeans(C.c_int(d), C.c_int64(n), _p(x), C.c_int64(k), C.c_int(niter),
                          C.c_uint64(seed), _p(cent))
    if rc != 0:
        raise RuntimeError(f"kmeans: need at least k={k} training points, got {n}")
    return cent


def merge(Dall, Iall):
    """float_maxheap_array_t semantics over S shards: Dall/Iall [S, nq, k]."""
    Dall, Iall = _f32(Dall), _i64(Iall)
    S, nq, k = Dall.shape
    outD = np.empty((nq, k), dtype=np.float32)
    outI = np.empty((nq, k), dtype=np.int64)
    lib().orc_merge(C.c_int64(S), C.c_int64(nq), C.c_int64(k), _p(Dall), _p(Iall), _p(outD), _p(outI))
    return outD, outI


# ---------------------------------------------------------------- index objects
class _OracleState:
    """get_state / set_state over the scalars and arrays engine.StateLayout lists for the oracle's kind;
    the arrays are attributes of the same names"""

    def get_state(self):
        lay = StateLayout(self)
        st = {"kind": self.kind, "d": self.d}
        st.update((key, getattr(self, key)) for key in lay.scalars)
        st.update((name, getattr(self, name)) for name in lay.arrays)
        return st

    def set_state(self, st):
        lay = StateLayout(self)
        for name in lay.arrays:
            if name != "tvals":  # recomputed (or taken) by OracleIVFPQ.set_state
                setattr(self, name, np.ascontiguousarray(st[name], dtype=STATE_ARRAYS[name][0]).reshape(lay.shape(name)))
        if "k_factor" in lay.scalars and "k_factor" in st:
            self.k_factor = float(st["k_factor"])


class _Quantizer:
    def __init__(self, owner):
        self._o = owner

    def reconstruct_n(self, i0, n):
        return self._o.centroids[i0:i0 + n].copy()


class OracleFlat(_OracleState):
    """faiss.IndexFlatIP / IndexFlatL2 restated (reference index.py:94, 25-33)."""

    kind = "flat"

    def __init__(self, d, metric=METRIC_IP):
        self.d, self.metric = int(d), int(metric)
        self.xb = np.zeros((0, self.d), dtype=np.float32)
        self.is_trained = True

    @property
    def ntotal(self):
        return self.xb.shape[0]

    def train(self, x):
        pass

    def add(self, x):
        self.xb = np.concatenate([self.xb, _f32(x)], axis=0)

    def search(self, x, k):
        return flat_search(self.metric, self.xb, x, k)

    def reconstruct_rows(self, ids):
        out = np.full((len(ids), self.d), np.nan, dtype=np.float32)
        ok = ids >= 0
        out[ok] = self.xb[ids[ok]]
        return out

    def search_and_reconstruct(self, x, k):
        D, I = self.search(x, k)
        R = self.reconstruct_rows(I.reshape(-1)).reshape(I.shape[0], I.shape[1], self.d)
        return D, I, R


class _OracleIVF(_OracleState):
    def __init__(self, d, nlist, coarse_metric):
        self.d, self.nlist, self.coarse_metric = int(d), int(nlist), int(coarse_metric)
        self.nprobe = 1  # faiss default
        self.centroids = None
        self.quantizer = _Quantizer(self)
        self.list_off = np.zeros(self.nlist + 1, dtype=np.int64)
        self.ids = np.zeros((0,), dtype=np.int64)
        self.ntotal = 0
        self.is_trained = False
        self.last_ndis = 0
        self.train_niter = 25
        self.train_seed = 1234

    # payload handling supplied by subclasses: _encode(x, list_of) -> dict of per-row arrays
    def _train_coarse(self, x):
        x = _f32(x)
        maxpts = 256 * self.nlist  # faiss Clustering: max_points_per_centroid = 256
        if x.shape[0] > maxpts:
            rs = np.random.RandomState(self.train_seed)
            x = x[rs.permutation(x.shape[0])[:maxpts]]
        self.centroids = kmeans(x, self.nlist, self.train_niter, self.train_seed)

    def add(self, x):
        x = _f32(x)
        n = x.shape[0]
        list_of = assign(self.coarse_metric, self.centroids, x)
        new_ids = np.arange(self.ntotal, self.ntotal + n, dtype=np.int64)
        rows = self._encode(x, list_of)
        # merge into list-sorted storage, ids ascending inside each list
        old_list = np.repeat(np.arange(self.nlist, dtype=np.int64), np.diff(self.list_off))
        all_list = np.concatenate([old_list, list_of])
        order = np.argsort(all_list, kind="stable")
        self.ids = np.concatenate([self.ids, new_ids])[order]
        for name, arr in rows.items():
            cur = getattr(self, name)
            setattr(self, name, np.concatenate([cur, arr], axis=0)[order])
        counts = np.bincount(all_list, minlength=self.nlist)
        self.list_off = np.concatenate([[0], np.cumsum(counts)]).astype(np.int64)
        self.ntotal += n

    def _eff_nprobe(self):
        return max(1, min(int(self.nprobe), self.nlist))

    def list_of_rows(self):
        return np.repeat(np.arange(self.nlist, dtype=np.int64), np.diff(self.list_off))

    def search_and_reconstruct(self, x, k):
        D, I = self.search(x, k)
        R = self.reconstruct_rows(I.reshape(-1)).reshape(I.shape[0], I.shape[1], self.d)
        return D, I, R

    def set_state(self, st):
        super().set_state(st)
        self.ntotal = int(self.ids.shape[0])
        self.is_trained = True


class OracleIVFFlat(_OracleIVF):
    """faiss.IndexIVFFlat restated (reference index.py:36-40 'ivf_simple')."""

    kind = "ivf_flat"

    def __init__(self, d, nlist, metric):
        super().__init__(d, nlist, metric)
        self.metric = int(metric)
        self.vecs = np.zeros((0, self.d), dtype=np.float32)

    def train(self, x):
        self._train_coarse(x)
        self.is_trained = True

    def _encode(self, x, list_of):
        return {"vecs": x}

    def search(self, x, k):
        x = _f32(x)
        nq = x.shape[0]
        D = np.empty((nq, k), dtype=np.float32)
        I = np.empty((nq, k), dtype=np.int64)
        nd = C.c_int64(0)
        lib().orc_ivfflat_search(C.c_int(self.metric), C.c_int(self.d), C.c_int64(self.nlist),
                                 _p(self.centroids), _p(self.list_off), _p(self.vecs), _p(self.ids),
                                 C.c_int64(nq), _p(x), C.c_int64(self._eff_nprobe()), C.c_int64(k),
                                 _p(D), _p(I), C.byref(nd))
        self.last_ndis = nd.value
        return D, I

    def reconstruct_rows(self, ids):
        inv = np.empty(self.ntotal, dtype=np.int64)
        inv[self.ids] = np.arange(self.ntotal)
        out = np.full((len(ids), self.d), np.nan, dtype=np.float32)
        ok = ids >= 0
        out[ok] = self.vecs[inv[ids[ok]]]
        return out


class OracleIVFPQ(_OracleIVF):
    """faiss.IndexIVFPQ(quantizer, d, nlist, M, nbits) restated: METRIC_L2,
    by_residual=True, precomputed-table decomposition (reference index.py:43-48)."""

    kind = "ivf_pq"

    def __init__(self, d, nlist, M, nbits=8, coarse_metric=METRIC_L2):
        super().__init__(d, nlist, coarse_metric)
        assert d % M == 0 and nbits <= 8
        self.M, self.ksub, self.dsub = int(M), 1 << int(nbits), d // M
        self.codebooks = None  # [M, ksub, dsub]
        self.codes = np.zeros((0, self.M), dtype=np.uint8)
        self.tvals = np.zeros((0,), dtype=np.float32)

    def train(self, x):
        x = _f32(x)
        self._train_coarse(x)
        # PQ trained on residuals of <= 256*ksub sampled training vectors (faiss)
        maxpts = 256 * self.ksub
        rs = np.random.RandomState(self.train_seed + 1)
        xs = x[rs.permutation(x.shape[0])[:maxpts]] if x.shape[0] > maxpts else x
        la = assign(self.coarse_metric, self.centroids, xs)
        res = xs - self.centroids[la]
        cb = np.empty((self.M, self.ksub, self.dsub), dtype=np.float32)
        for m in range(self.M):
            cb[m] = kmeans(res[:, m * self.dsub:(m + 1) * self.dsub], self.ksub, self.train_niter,
                           self.train_seed + 2 + m)
        self.codebooks = cb
        self.is_trained = True

    def _encode(self, x, list_of):
        n = x.shape[0]
        codes = np.empty((n, self.M), dtype=np.uint8)
        lib().orc_pq_encode(C.c_int(self.d), C.c_int(self.M), C.c_int(self.ksub), _p(self.codebooks),
                            _p(self.centroids), _p(list_of), _p(x), C.c_int64(n), _p(codes))
        return {"codes": codes, "tvals": self.compute_tvals(codes, list_of)}

    def compute_tvals(self, codes, list_of):
        codes = np.ascontiguousarray(codes, dtype=np.uint8)
        list_of = _i64(list_of)
        t = np.empty((codes.shape[0],), dtype=np.float32)
        lib().orc_pq_tvals(C.c_int(self.d), C.c_int(self.M), C.c_int(self.ksub), _p(self.codebooks),
                           _p(self.centroids), _p(list_of), _p(codes), C.c_int64(codes.shape[0]), _p(t))
        return t

    def query_lut(self, q):
        q = _f32(q)
        lut = np.empty((self.M, self.ksub), dtype=np.float32)
        lib().orc_pq_query_lut(C.c_int(self.d), C.c_int(self.M), C.c_int(self.ksub),
                               _p(self.codebooks), _p(q), _p(lut))
        return lut

    def search(self, x, k):
        x = _f32(x)
        nq = x.shape[0]
        D = np.empty((nq, k), dtype=np.float32)
        I = np.empty((nq, k), dtype=np.int64)
        nd = C.c_int64(0)
        lib().orc_ivfpq_search(C.c_int(self.coarse_metric), C.c_int(self.d), C.c_int64(self.nlist),
                               _p(self.centroids), C.c_int(self.M), C.c_int(self.ksub),
                               _p(self.codebooks), _p(self.list_off), _p(self.codes), _p(self.tvals),
                               _p(self.ids), C.c_int64(nq), _p(x), C.c_int64(self._eff_nprobe()),
                               C.c_int64(k), _p(D), _p(I), C.byref(nd))
        self.last_ndis = nd.value
        return D, I

    def reconstruct_rows(self, ids):
        inv = np.empty(self.ntotal, dtype=np.int64)
        inv[self.ids] = np.arange(self.ntotal)
        lo = self.list_of_rows()
        out = np.full((len(ids), self.d), np.nan, dtype=np.float32)
        for r, i in enumerate(ids):
            if i < 0:
                continue
            pos = inv[i]
            v = self.centroids[lo[pos]].copy()
            for m in range(self.M):
                v[m * self.dsub:(m + 1) * self.dsub] += self.codebooks[m, self.codes[pos, m]]
            out[r] = v
        return out

    def set_state(self, st, recompute_tvals=True):
        super().set_state(st)
        if recompute_tvals or "tvals" not in st:
            self.tvals = self.compute_tvals(self.codes, self.list_of_rows())
        else:
            self.tvals = _f32(st["tvals"])


class OracleIVFSQ(_OracleIVF):
    """faiss.IndexIVFScalarQuantizer(quantizer, d, nlist, QT_fp16) restated:
    METRIC_L2, by_residual=True (reference index.py:63-68)."""

    kind = "ivf_sq"

    def __init__(self, d, nlist, coarse_metric=METRIC_L2):
        super().__init__(d, nlist, coarse_metric)
        self.codes16 = np.zeros((0, self.d), dtype=np.uint16)

    def train(self, x):
        self._train_coarse(x)
        self.is_trained = True

    def _encode(self, x, list_of):
        n = x.shape[0]
        codes = np.empty((n, self.d), dtype=np.uint16)
        lib().orc_sq_encode(C.c_int(self.d), _p(self.centroids), _p(list_of), _p(x), C.c_int64(n),
                            _p(codes))
        return {"codes16": codes}

    def search(self, x, k):
        x = _f32(x)
        nq = x.shape[0]
        D = np.empty((nq, k), dtype=np.float32)
        I = np.empty((nq, k), dtype=np.int64)
        nd = C.c_int64(0)
        lib().orc_ivfsq_search(C.c_int(self.coarse_metric), C.c_int(self.d), C.c_int64(self.nlist),
                               _p(self.centroids), _p(self.list_off), _p(self.codes16), _p(self.ids),
                               C.c_int64(nq), _p(x), C.c_int64(self._eff_nprobe()), C.c_int64(k),
                               _p(D), _p(I), C.byref(nd))
        self.last_ndis = nd.value
        return D, I

    def reconstruct_rows(self, ids):
        inv = np.empty(self.ntotal, dtype=np.int64)
        inv[self.ids] = np.arange(self.ntotal)
        lo = self.list_of_rows()
        out = np.full((len(ids), self.d), np.nan, dtype=np.float32)
        ok = ids >= 0
        pos = inv[ids[ok]]
        out[ok] = self.centroids[lo[pos]] + half_to_float(self.codes16[pos])
        return out


def make_index(kind, d, metric=METRIC_IP, nlist=0, M=0, nbits=8):
    """Same (kind, metric) meaning as the product's engine factory."""
    if kind == "flat":
        return OracleFlat(d, metric)
    if kind == "ivf_flat":
        return OracleIVFFlat(d, nlist, metric)
    if kind == "ivf_pq":
        return OracleIVFPQ(d, nlist, M, nbits, coarse_metric=metric)
    if kind == "ivf_sq":
        return OracleIVFSQ(d, nlist, coarse_metric=metric)
    raise ValueError(kind)
