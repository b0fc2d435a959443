"""CPU oracle of the "PQ{M}" shard (faiss IndexPQ(d, M, 8, metric) without lists; test infrastructure --
NOT product code).  The arithmetic is the canonical one of DESIGN.md section 2:

  train   sub-quantizer m = kmeans(column slice m of the first min(n, 256 * 256) rows, 256, niter,
          train_seed + 1 + m), the device build's k-means (tests/oracle_train.kmeans)
  encode  code_m = argmin_j l2_seq(x_m, P[m][j]), ties -> the smaller j
  table   L2: LUT[m][j] = l2_seq(q_m, P[m][j]) (df = q - p; acc = fmaf(df, df, acc), t ascending from +0);
          IP: LUT[m][j] = -ip_seq(q_m, P[m][j]) (acc = fmaf(q, p, acc), then negated)
  value   the halving tree over LUT[m][code_m], padded with +0 to the next power of two
  output  ranked by (value, id); D = value (L2) or -value (IP); missing: (+FLT_MAX, -1) / (-FLT_MAX, -1)
  recon   P[m][code_m]

numpy float32 with the correctly rounded fmaf of tests/oracle_sq8.fma32, so every value is the one the CUDA
kernels compute.  The state is the engine's: "metric", "M", "ksub", "codebooks" and "codes"."""
import numpy as np

from distributed_faiss_b200.index import factory_spec
from oracle import oracle as O
from tests.oracle_sq8 import fma32

KSUB = 256
TRAIN_ROWS = 256 * KSUB
F32 = np.float32
FLT_MAX = np.finfo(np.float32).max


def tables(codebooks, x, metric):
    """LUT f32[n, M, 256] of rows x f32[n, d]"""
    M, ksub, dsub = codebooks.shape
    x = np.ascontiguousarray(x, dtype=F32).reshape(-1, M, 1, dsub)
    acc = np.zeros((x.shape[0], M, ksub), dtype=F32)
    for t in range(dsub):
        if metric == O.METRIC_L2:
            df = (x[..., t] - codebooks[None, :, :, t]).astype(F32)
            acc = fma32(df, df, acc)
        else:
            acc = fma32(x[..., t], codebooks[None, :, :, t], acc)
    return acc if metric == O.METRIC_L2 else (-acc).astype(F32)


def encode(codebooks, x, chunk=2048):
    """codes u8[n, M]: the nearest sub-centroid of every sub-vector, ties -> the smaller index"""
    x = np.ascontiguousarray(x, dtype=F32)
    out = np.empty((x.shape[0], codebooks.shape[0]), dtype=np.uint8)
    for i in range(0, x.shape[0], chunk):
        out[i:i + chunk] = np.argmin(tables(codebooks, x[i:i + chunk], O.METRIC_L2), axis=2)
    return out


def pq_sum(vals):
    """the halving tree over the last axis of vals f32[..., M], padded with +0 to the next power of two"""
    vals = np.asarray(vals, dtype=F32)
    M = vals.shape[-1]
    P = 1
    while P < M:
        P *= 2
    v = np.zeros(vals.shape[:-1] + (P,), dtype=F32)
    v[..., :M] = vals
    off = P // 2
    while off >= 1:
        v[..., :off] = (v[..., :off] + v[..., off:2 * off]).astype(F32)
        off //= 2
    return v[..., 0]


def _key(v):
    """the composite key of dfx_f2key: -0 -> +0, then order-preserving uint32"""
    u = (np.asarray(v, dtype=F32) + F32(0)).view(np.uint32).astype(np.uint64)
    return np.where(u & 0x80000000, (~u) & 0xFFFFFFFF, u | 0x80000000)


def _key2f(k):
    k = np.asarray(k, dtype=np.uint64)
    u = np.where(k & 0x80000000, k & 0x7FFFFFFF, (~k) & 0xFFFFFFFF).astype(np.uint32)
    return u.view(F32)


class OracleFlatPQ(O._OracleState):
    """faiss.IndexPQ(d, M, 8, metric) (the factory strings "PQ{M}" / "PQ{M}x8")"""

    kind = "flat_pq"

    def __init__(self, d, M, metric=O.METRIC_IP):
        assert d % M == 0 and M % 4 == 0
        self.d, self.M, self.metric = int(d), int(M), int(metric)
        self.ksub, self.dsub = KSUB, self.d // self.M
        self.codebooks = None  # [M, 256, dsub]
        self.codes = np.zeros((0, self.M), dtype=np.uint8)
        self.is_trained = False
        self.train_niter, self.train_seed = 25, 1234

    @property
    def ntotal(self):
        return self.codes.shape[0]

    def train(self, x):
        from tests.oracle_train import kmeans

        xs = np.ascontiguousarray(x, dtype=F32)[:TRAIN_ROWS]
        if xs.shape[0] < KSUB:
            raise RuntimeError(f"train: need at least {KSUB} vectors for PQ")
        self.codebooks = np.stack([kmeans(xs[:, m * self.dsub:(m + 1) * self.dsub], KSUB, self.train_niter,
                                          self.train_seed + 1 + m) for m in range(self.M)])
        self.codes = np.zeros((0, self.M), dtype=np.uint8)
        self.is_trained = True

    def add(self, x):
        assert self.is_trained, "add: index is not trained"
        self.codes = np.concatenate([self.codes, encode(self.codebooks, x)], axis=0)

    def set_state(self, st):
        super().set_state(st)
        self.is_trained = True

    def values(self, xq):
        """ranking values f32[nq, ntotal]"""
        lut = tables(self.codebooks, xq, self.metric)
        mi = np.arange(self.M)
        return np.stack([pq_sum(lut[q][mi[None, :], self.codes]) for q in range(lut.shape[0])])

    def search(self, x, k, chunk=64):
        x = np.ascontiguousarray(x, dtype=F32).reshape(-1, self.d)
        nq, n = x.shape[0], self.ntotal
        ip = self.metric == O.METRIC_IP
        D = np.full((nq, k), -FLT_MAX if ip else FLT_MAX, dtype=F32)
        I = np.full((nq, k), -1, dtype=np.int64)
        if n == 0:
            return D, I
        ids = np.arange(n, dtype=np.uint64)
        kk = min(k, n)
        for q0 in range(0, nq, chunk):
            comp = (_key(self.values(x[q0:q0 + chunk])) << np.uint64(32)) | ids[None, :]
            part = np.partition(comp, kk - 1, axis=1)[:, :kk] if kk < n else comp
            best = np.sort(part, axis=1)[:, :kk]
            v = _key2f(best >> np.uint64(32))
            D[q0:q0 + chunk, :kk] = -v if ip else v
            I[q0:q0 + chunk, :kk] = (best & np.uint64(0xFFFFFFFF)).astype(np.int64)
        return D, I

    def reconstruct_rows(self, ids):
        ids = np.asarray(ids, dtype=np.int64)
        out = np.full((len(ids), self.d), np.nan, dtype=F32)
        ok = ids >= 0
        out[ok] = self.codebooks[np.arange(self.M)[None, :], self.codes[ids[ok]]].reshape(-1, self.d)
        return out

    def search_and_reconstruct(self, x, k):
        D, I = self.search(x, k)
        return D, I, self.reconstruct_rows(I.reshape(-1)).reshape(I.shape[0], I.shape[1], self.d)


def flat_pq_engine_factory(cfg):
    """tests/oracle_flat_sq16.flat_sq16_engine_factory plus the factory strings "PQ{M}" / "PQ{M}x8", as
    distributed_faiss_b200.index.default_engine_factory builds them"""
    from tests.oracle_flat_sq16 import flat_sq16_engine_factory

    spec = factory_spec(cfg)
    if spec is not None and spec.kind == "flat_pq":
        return OracleFlatPQ(cfg.dim, spec.pq_m, spec.metric)
    return flat_sq16_engine_factory(cfg)
