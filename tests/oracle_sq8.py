"""CPU oracle of the IVF-SQ8 kind (test infrastructure -- NOT product code).

faiss.IndexIVFScalarQuantizer(quantizer, d, nlist, QT_8bit) restated: METRIC_L2, by_residual,
the non-uniform 8-bit codec trained by min-max (RS_minmax).  The arithmetic is the canonical one of
DESIGN.md section 2 [faiss-upstream: restated from knowledge of faiss impl/ScalarQuantizer.cpp,
not checked against faiss here]:

  train   r = x - c(assign(x)) over the first min(nt, 100000) rows of the k-means sample;
          vmin[i] = min r_i, vdiff[i] = max r_i - vmin[i]; trained = [vmin, vdiff]
  encode  t = vdiff[i] != 0 ? (r_i - vmin[i]) / vdiff[i] : 0, clamped to [0, 1];
          code = (int)(255 t), truncated
  decode  t = fmaf(code, 1/255, 0.5/255);  x = fmaf(t, vdiff[i], vmin[i])   (faiss's AVX2 form)
  search  rq = q - c;  dist = sum_i (rq_i - x_i)^2 in the warp-dot order
  recon   c + x

It builds on the existing CPU oracle (oracle/oracle.py): the coarse quantizer, k-means and
assignment are its functions, and the list scan is its IVF-Flat L2 scan (`orc_ivfflat_search`,
warp-dot order) run on the residual query against the decoded rows -- the SQ8 distance is exactly
that scan's distance once the rows are decoded.  Only the codec is new here, in numpy float32
with a correctly rounded fmaf (`fma32`), so every value is the one the CUDA kernels compute.
"""
import ctypes as C

import numpy as np

from oracle import oracle as O
from oracle import ref_numpy as R

SQ8_SCALE = np.float32(1) / np.float32(255)
SQ8_BIAS = np.float32(0.5) / np.float32(255)
TRAIN_ROWS = 100_000  # faiss ScalarQuantizer trains on at most this many rows


def fma32(a, b, c):
    """fmaf(a, b, c) on float32 arrays, correctly rounded: a*b is exact in float64, a + c is
    rounded to odd in float64 (exact error by TwoSum), and rounding that to float32 is then the
    correctly rounded result (53 >= 2 * 24 + 2)."""
    a = np.asarray(a, dtype=np.float32).astype(np.float64)
    b = np.asarray(b, dtype=np.float32).astype(np.float64)
    c = np.asarray(c, dtype=np.float32).astype(np.float64)
    p = a * b
    s = p + c
    bb = s - p
    err = (p - (s - bb)) + (c - bb)
    even = (s.view(np.int64) & 1) == 0
    fix = (err != 0) & even
    if np.any(fix):
        s = np.where(fix, np.nextafter(s, np.where(err > 0, np.inf, -np.inf)), s)
    return s.astype(np.float32)


def sq8_train(centroids, xt, coarse_metric):
    """trained f32[2, d] = [vmin, vdiff] from the residuals of the first TRAIN_ROWS rows of xt"""
    xs = np.ascontiguousarray(xt[:TRAIN_ROWS], dtype=np.float32)
    res = xs - centroids[O.assign(coarse_metric, centroids, xs)]
    vmin = res.min(axis=0)
    return np.stack([vmin, res.max(axis=0) - vmin]).astype(np.float32)


def sq8_encode_residuals(trained, r):
    r = np.asarray(r, dtype=np.float32)
    vmin, vdiff = trained[0], trained[1]
    nz = vdiff != 0
    with np.errstate(divide="ignore", invalid="ignore"):
        t = np.where(nz, (r - vmin) / np.where(nz, vdiff, np.float32(1)), np.float32(0)).astype(np.float32)
    t = np.minimum(np.maximum(t, np.float32(0)), np.float32(1))
    return (np.float32(255) * t).astype(np.int32).astype(np.uint8)


def sq8_encode(trained, centroids, list_of, x):
    x = np.asarray(x, dtype=np.float32)
    return sq8_encode_residuals(trained, x - centroids[np.asarray(list_of, dtype=np.int64)])


_T_OF_CODE = None


def sq8_decode(trained, codes):
    """decoded residuals f32[n, d] of codes u8[n, d]"""
    global _T_OF_CODE
    if _T_OF_CODE is None:
        _T_OF_CODE = fma32(np.arange(256, dtype=np.float32), SQ8_SCALE, SQ8_BIAS)
    t = _T_OF_CODE[np.asarray(codes, dtype=np.uint8)]
    return fma32(t, trained[1][None, :], trained[0][None, :])


class OracleIVFSQ8(O._OracleIVF):
    """faiss.IndexIVFScalarQuantizer(quantizer, d, nlist, QT_8bit) restated: METRIC_L2,
    by_residual (the factory string "IVF{n},SQ8")."""

    kind = "ivf_sq8"

    def __init__(self, d, nlist, coarse_metric=O.METRIC_L2):
        super().__init__(d, nlist, coarse_metric)
        self.sq_trained = None
        self.codes8 = np.zeros((0, self.d), dtype=np.uint8)

    def train(self, x):
        x = np.ascontiguousarray(x, dtype=np.float32)
        maxpts = 256 * self.nlist  # the sample of _OracleIVF._train_coarse
        if x.shape[0] > maxpts:
            rs = np.random.RandomState(self.train_seed)
            x = x[rs.permutation(x.shape[0])[:maxpts]]
        self.centroids = O.kmeans(x, self.nlist, self.train_niter, self.train_seed)
        self.sq_trained = sq8_train(self.centroids, x, self.coarse_metric)
        self.is_trained = True

    def _encode(self, x, list_of):
        return {"codes8": sq8_encode(self.sq_trained, self.centroids, list_of, x)}

    def search(self, x, k):
        x = np.ascontiguousarray(x, dtype=np.float32)
        nq, d = x.shape
        nprobe = self._eff_nprobe()
        keys, _ = O.coarse(self.coarse_metric, self.centroids, x, nprobe)
        cand_D = [[] for _ in range(nq)]
        cand_I = [[] for _ in range(nq)]
        ndis = 0
        dummy = np.zeros((1, d), dtype=np.float32)
        for l in np.unique(keys[keys >= 0]):
            a, b = int(self.list_off[l]), int(self.list_off[l + 1])
            qs = np.nonzero((keys == l).any(axis=1))[0]
            ndis += (b - a) * len(qs)
            if b == a:
                continue
            rq = np.ascontiguousarray(x[qs] - self.centroids[l], dtype=np.float32)
            xhat = np.ascontiguousarray(sq8_decode(self.sq_trained, self.codes8[a:b]))
            ids = np.ascontiguousarray(self.ids[a:b], dtype=np.int64)
            kk = min(k, b - a)
            D = np.empty((len(qs), kk), dtype=np.float32)
            I = np.empty((len(qs), kk), dtype=np.int64)
            nd = C.c_int64(0)
            # the IVF-Flat L2 scan of ONE list holding the decoded rows: warp-dot sum of (rq - x)^2
            O.lib().orc_ivfflat_search(C.c_int(O.METRIC_L2), C.c_int(d), C.c_int64(1), O._p(dummy),
                                       O._p(np.array([0, b - a], dtype=np.int64)), O._p(xhat), O._p(ids),
                                       C.c_int64(len(qs)), O._p(rq), C.c_int64(1), C.c_int64(kk),
                                       O._p(D), O._p(I), C.byref(nd))
            for j, qi in enumerate(qs):
                cand_D[qi].append(D[j])
                cand_I[qi].append(I[j])
        outD = np.full((nq, k), O.FLT_MAX, dtype=np.float32)
        outI = np.full((nq, k), -1, dtype=np.int64)
        for qi in range(nq):
            if not cand_D[qi]:
                continue
            v, ids = np.concatenate(cand_D[qi]), np.concatenate(cand_I[qi])
            order = np.lexsort((ids, v))[:k]  # total order (value asc, id asc)
            outD[qi, :len(order)] = v[order]
            outI[qi, :len(order)] = ids[order]
        self.last_ndis = ndis
        return outD, outI

    def reconstruct_rows(self, ids):
        ids = np.asarray(ids, dtype=np.int64)
        inv = np.empty(self.ntotal, dtype=np.int64)
        inv[self.ids] = np.arange(self.ntotal)
        lo = self.list_of_rows()
        out = np.full((len(ids), self.d), np.nan, dtype=np.float32)
        ok = ids >= 0
        pos = inv[ids[ok]]
        out[ok] = self.centroids[lo[pos]] + sq8_decode(self.sq_trained, self.codes8[pos])
        return out


def make_index(kind, d, metric=O.METRIC_IP, nlist=0, M=0, nbits=8):
    """oracle.make_index plus "ivf_sq8" (same (kind, metric) meaning as the engine factory)"""
    if kind == "ivf_sq8":
        return OracleIVFSQ8(d, nlist, coarse_metric=metric)
    return O.make_index(kind, d, metric=metric, nlist=nlist, M=M, nbits=nbits)


# ---------------------------------------------------------------- float64 restatement
def reconstruct_all_f64(state):
    """float64 decode of every stored vector, list-sorted order: c + vmin + (code + 0.5) / 255 * vdiff"""
    list_of = np.repeat(np.arange(state["nlist"]), np.diff(state["list_off"]))
    tr = np.asarray(state["sq_trained"], dtype=np.float64)
    t = (np.asarray(state["codes8"], dtype=np.float64) + 0.5) / 255.0
    return state["centroids"].astype(np.float64)[list_of] + tr[0] + t * tr[1]


def ivf_sq8_search_f64(state, xq, nprobe, k):
    """ref_numpy.ivf_search for the SQ8 kind: float64 distances from the float64 decode"""
    keys = R.coarse(state["coarse_metric"], state["centroids"], xq, nprobe)
    recon = reconstruct_all_f64(state)
    off = state["list_off"]
    D = np.empty((xq.shape[0], k))
    I = np.empty((xq.shape[0], k), dtype=np.int64)
    for i in range(xq.shape[0]):
        rows = np.concatenate([np.arange(off[l], off[l + 1]) for l in keys[i]] + [np.zeros(0, np.int64)]).astype(np.int64)
        D[i], I[i] = R._topk(R._values(R.METRIC_L2, xq[i], recon[rows]), state["ids"][rows], k, R.METRIC_L2)
    return D, I


# ---------------------------------------------------------------- oracle-backed engine factory
def oracle_engine_factory(cfg):
    """tests/oracle_engine.oracle_engine_factory plus the factory-string paths of
    distributed_faiss_b200.index.default_engine_factory, through the same parser"""
    from distributed_faiss_b200.index import factory_spec
    from tests.oracle_engine import oracle_engine_factory as builders

    spec = factory_spec(cfg)
    if spec is None:
        return builders(cfg)
    ix = make_index(spec.kind, cfg.dim, metric=spec.metric, nlist=spec.nlist, M=spec.pq_m)
    if cfg.index_builder_type == "ivf_gpu":
        ix.nprobe = cfg.nprobe
    return ix
