"""CPU oracle of the IVF-PQ FastScan kind (test infrastructure -- NOT product code).

faiss.index_factory(d, "IVF{n},PQ{M}x4fs") restated: IndexIVFPQFastScan with nbits = 4, METRIC_L2 and
by_residual = false.  The arithmetic is the canonical one of DESIGN.md section 2 [faiss-upstream:
restated from knowledge of faiss IndexIVFPQFastScan.cpp, IndexIVFFastScan.cpp and
utils/quantize_lut.cpp, not checked against faiss here]:

  train   coarse k-means as the other IVF kinds; the 16-centroid sub-quantizers on the RAW
          sub-vectors of the first min(nt, 256 * 16) rows of the k-means sample
  encode  code_m = argmin_j l2_seq(x_m, P[m][j]), ties -> smaller j (no residual, no t-value)
  table   LUT[m][j] = l2_seq(q_m, P[m][j])  (df = q - p; acc = fmaf(df, df, acc), t ascending)
  quant   mn_m = min_j LUT, span_m = max_j LUT - mn_m; a = min(255 / max_m span_m, 65535 / sum_m span_m)
          (a = 1 when the sum is 0); b = sum_m mn_m (fp32, m ascending from +0);
          LUTq = floorf(fmaf(LUT - mn_m, a, 0.5f))
  scan    acc = sum_m LUTq[m][code_m], an exact integer; ranked by (acc, id)
  output  D = fmaf((float)acc, 1 / a, b)
  recon   P[m][code_m] (no centroid)

numpy float32 with a correctly rounded fmaf (tests/oracle_sq8.fma32), so every value is the one the
CUDA kernels compute.  The coarse quantizer, k-means and assignment are those of oracle/oracle.py.
"""
import numpy as np

from oracle import oracle as O
from tests.oracle_sq8 import fma32

KSUB = 16
TRAIN_ROWS = 256 * KSUB
F32 = np.float32


def l2_tables(codebooks, x):
    """LUT f32[n, M, 16] = l2_seq(x_m, P[m][j]) of rows x f32[n, d] (the order of encode and search)"""
    M, ksub, dsub = codebooks.shape
    x = np.ascontiguousarray(x, dtype=F32).reshape(-1, M, 1, dsub)
    acc = np.zeros((x.shape[0], M, ksub), dtype=F32)
    for t in range(dsub):
        df = (x[..., t] - codebooks[None, :, :, t]).astype(F32)
        acc = fma32(df, df, acc)
    return acc


def encode(codebooks, x, chunk=2048):
    """codes u8[n, M]: the nearest sub-centroid of every sub-vector, ties -> the smaller index"""
    x = np.ascontiguousarray(x, dtype=F32)
    out = np.empty((x.shape[0], codebooks.shape[0]), dtype=np.uint8)
    for i in range(0, x.shape[0], chunk):
        out[i:i + chunk] = np.argmin(l2_tables(codebooks, x[i:i + chunk]), axis=2)
    return out


def quantize_tables(lut):
    """lut f32[nq, M, 16] -> (LUTq u8[nq, M, 16], a f32[nq], b f32[nq], 1 / a f32[nq])"""
    lut = np.asarray(lut, dtype=F32)
    nq, M, _ = lut.shape
    mn = lut.min(axis=2)
    span = (lut.max(axis=2) - mn).astype(F32)
    span_max = span.max(axis=1)
    span_sum = np.zeros(nq, dtype=F32)
    b = np.zeros(nq, dtype=F32)
    for m in range(M):                       # fp32, m ascending from +0
        span_sum = (span_sum + span[:, m]).astype(F32)
        b = (b + mn[:, m]).astype(F32)
    flat = span_sum == 0
    with np.errstate(divide="ignore", invalid="ignore"):
        a = np.minimum(F32(255) / span_max, F32(65535) / span_sum).astype(F32)
    a = np.where(flat, F32(1), a).astype(F32)
    diff = (lut - mn[:, :, None]).astype(F32)
    lutq = np.floor(fma32(diff, a[:, None, None], F32(0.5))).astype(np.uint8)
    return lutq, a, b, (F32(1) / a).astype(F32)


class OracleIVFPQFastScan(O._OracleIVF):
    """faiss.IndexIVFPQFastScan(quantizer, d, nlist, M, 4), by_residual = false (the factory string
    "IVF{n},PQ{M}x4fs")"""

    kind = "ivf_pq_fs"

    def __init__(self, d, nlist, M, coarse_metric=O.METRIC_L2):
        super().__init__(d, nlist, coarse_metric)
        assert d % M == 0 and M % 8 == 0
        self.M, self.ksub, self.dsub = int(M), KSUB, d // int(M)
        self.codebooks = None  # [M, 16, dsub]
        self.codes = np.zeros((0, self.M), dtype=np.uint8)

    def train(self, x):
        x = np.ascontiguousarray(x, dtype=F32)
        maxpts = 256 * self.nlist  # the sample of _OracleIVF._train_coarse
        if x.shape[0] > maxpts:
            rs = np.random.RandomState(self.train_seed)
            x = x[rs.permutation(x.shape[0])[:maxpts]]
        self.centroids = O.kmeans(x, self.nlist, self.train_niter, self.train_seed)
        xs = x[:TRAIN_ROWS]
        cb = np.empty((self.M, KSUB, self.dsub), dtype=F32)
        for m in range(self.M):
            cb[m] = O.kmeans(xs[:, m * self.dsub:(m + 1) * self.dsub], KSUB, self.train_niter, self.train_seed + 1 + m)
        self.codebooks = cb
        self.is_trained = True

    def _encode(self, x, list_of):
        return {"codes": encode(self.codebooks, x)}

    def query_tables(self, x):
        """(LUTq, a, b, 1 / a) of queries x"""
        return quantize_tables(l2_tables(self.codebooks, x))

    def search(self, x, k):
        x = np.ascontiguousarray(x, dtype=F32)
        nq = x.shape[0]
        keys, _ = O.coarse(self.coarse_metric, self.centroids, x, self._eff_nprobe())
        lutq, _, b, one_a = self.query_tables(x)
        outD = np.full((nq, k), O.FLT_MAX, dtype=F32)
        outI = np.full((nq, k), -1, dtype=np.int64)
        ndis = 0
        mi = np.arange(self.M)
        for q in range(nq):
            rows = [np.arange(self.list_off[l], self.list_off[l + 1]) for l in keys[q] if l >= 0]
            rows = np.concatenate(rows + [np.zeros(0, np.int64)]).astype(np.int64)
            ndis += len(rows)
            if len(rows) == 0:
                continue
            acc = lutq[q][mi[None, :], self.codes[rows]].astype(np.int64).sum(axis=1)
            ids = self.ids[rows]
            order = np.lexsort((ids, acc))[:k]  # total order (acc asc, id asc)
            outD[q, :len(order)] = fma32(acc[order].astype(F32), one_a[q], b[q])
            outI[q, :len(order)] = ids[order]
        self.last_ndis = ndis
        return outD, outI

    def reconstruct_rows(self, ids):
        ids = np.asarray(ids, dtype=np.int64)
        inv = np.empty(self.ntotal, dtype=np.int64)
        inv[self.ids] = np.arange(self.ntotal)
        out = np.full((len(ids), self.d), np.nan, dtype=F32)
        ok = ids >= 0
        codes = self.codes[inv[ids[ok]]]
        out[ok] = self.codebooks[np.arange(self.M)[None, :], codes].reshape(-1, self.d)
        return out


def make_index(kind, d, metric=O.METRIC_IP, nlist=0, M=0, nbits=8):
    """tests/oracle_sq8.make_index plus "ivf_pq_fs" (metric: the coarse quantizer's, L2)"""
    from tests.oracle_sq8 import make_index as others

    if kind == "ivf_pq_fs":
        return OracleIVFPQFastScan(d, nlist, M, coarse_metric=metric)
    return others(kind, d, metric=metric, nlist=nlist, M=M, nbits=nbits)


def oracle_engine_factory(cfg):
    """tests/oracle_sq8.oracle_engine_factory plus the "IVF{n},PQ{M}x4fs" factory strings, through the
    parser of distributed_faiss_b200.index.default_engine_factory"""
    from distributed_faiss_b200.index import factory_spec
    from tests.oracle_sq8 import oracle_engine_factory as others

    spec = factory_spec(cfg)
    if spec is None or spec.kind != "ivf_pq_fs":
        return others(cfg)
    ix = OracleIVFPQFastScan(cfg.dim, spec.nlist, spec.pq_m, coarse_metric=spec.metric)
    if cfg.index_builder_type == "ivf_gpu":
        ix.nprobe = cfg.nprobe
    return ix


# ---------------------------------------------------------------- float64 restatement
def adc_f64(state, xq, rows):
    """float64 |q - x_hat|^2 of queries xq [nq, d] against the stored rows `rows` (positions in the
    list-sorted storage): [nq, len(rows)]"""
    cb = np.asarray(state["codebooks"], dtype=np.float64)
    M = cb.shape[0]
    xhat = cb[np.arange(M)[None, :], np.asarray(state["codes"])[rows]].reshape(len(rows), -1)
    q = np.asarray(xq, dtype=np.float64)
    return ((q[:, None, :] - xhat[None, :, :]) ** 2).sum(axis=2)


def dequant_bound(M, a):
    """|D - |q - x_hat|^2| <= (M / 2 + 1) / a: every table entry is rounded to the nearest 1 / a, and the
    +1 covers the fp32 rounding of 1 / a and of the output fmaf"""
    return (M / 2 + 1) / np.asarray(a, dtype=np.float64)
