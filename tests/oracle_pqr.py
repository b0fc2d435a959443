"""CPU oracle of the IVF-PQR kind (test infrastructure -- NOT product code).

faiss.index_factory(d, "IVF{n},PQ{M}+{M2}") restated: IndexIVFPQR(quantizer, d, nlist, M, 8, M2, 8),
METRIC_L2, by_residual, k_factor = 4.  The arithmetic is the canonical one of DESIGN.md section 2
[faiss-upstream: restated from knowledge of faiss IndexIVFPQR.cpp, not checked against faiss here]:

  train   as IVF-PQ; then on the same training residuals r: r2 = r - decode(encode(r)), and the
          refinement PQ (M2 sub-quantizers of 256 centroids) is trained on r2
  add     list, codes and t-value as IVF-PQ; r2 = (x - c) - P1[m][code_m] (one fp32 rounding per
          subtraction); refine_codes[id] = argmin_j l2_seq(r2_m2, P2[m2][j]), ties -> smaller j,
          stored by id (arrival order), outside the lists
  search  k' = (int64)((float)k * k_factor); the IVF-PQ search for k' candidates (oracle.OracleIVFPQ);
          for each candidate, dimension i: r1 = q_i - c_i, r2 = r1 - P1[.], df = P2[.] - r2,
          acc = fmaf(df, df, acc) in the warp-dot order (oracle.warp_dot, mode 1); the k smallest
          under the total order (dis, id), padded with (FLT_MAX, -1)
  recon   (c + P1[m][code_m]) + P2[m2][refine_code_m2]

numpy float32 with a correctly rounded fmaf (tests/oracle_sq8.fma32), so every value is the one the
CUDA kernels compute.  The first stage, the coarse quantizer, k-means and assignment are those of
oracle/oracle.py.
"""
import ctypes as C

import numpy as np

from oracle import oracle as O
from tests.oracle_sq8 import fma32

F32 = np.float32
KSUB = 256
K_MAX = 16384  # the most candidates a search re-ranks


def first_stage_k(k, k_factor):
    """k' = (int64)(k * k_factor), the product in fp32 as faiss computes it"""
    return int(F32(k) * F32(k_factor))


def warp_l2(df):
    """sum_i df_i^2 of the rows of df f32[n, d] in the warp-dot order: lane j accumulates
    fmaf(df, df, acc) over k = 128 t + 4 j + u, then the butterfly xor 16 .. 1.  The row is padded
    with zeros to whole 128-wide steps: fmaf(0, 0, acc) == acc."""
    df = np.ascontiguousarray(df, dtype=F32)
    n, d = df.shape
    pad = np.zeros((n, -(-d // 128) * 128), dtype=F32)
    pad[:, :d] = df
    steps = pad.reshape(n, -1, 32, 4)
    acc = np.zeros((n, 32), dtype=F32)
    for t in range(steps.shape[1]):
        for u in range(4):
            v = steps[:, t, :, u]
            acc = fma32(v, v, acc)
    lanes = np.arange(32)
    for off in (16, 8, 4, 2, 1):
        acc = (acc + acc[:, lanes ^ off]).astype(F32)
    return acc[:, 0]


def encode(codebooks, x):
    """codes u8[n, M] of the rows x themselves: code_m = argmin_j l2_seq(x_m, P[m][j]), ties -> the
    smaller j (the C oracle's IVF-PQ encode against one all-zero centroid: x - 0 == x)"""
    x = np.ascontiguousarray(x, dtype=F32)
    M, ksub, _ = codebooks.shape
    n, d = x.shape
    out = np.empty((n, M), dtype=np.uint8)
    O.lib().orc_pq_encode(C.c_int(d), C.c_int(M), C.c_int(ksub), O._p(np.ascontiguousarray(codebooks, dtype=F32)),
                          O._p(np.zeros((1, d), dtype=F32)), O._p(np.zeros(n, dtype=np.int64)), O._p(x),
                          C.c_int64(n), O._p(out))
    return out


def decode(codebooks, codes):
    """f32[n, d] = P[m][code_m] side by side"""
    M = codebooks.shape[0]
    return codebooks[np.arange(M)[None, :], np.asarray(codes, dtype=np.int64)].reshape(len(codes), -1)


class OracleIVFPQR(O.OracleIVFPQ):
    """faiss.IndexIVFPQR(quantizer, d, nlist, M, 8, M2, 8) (the factory string "IVF{n},PQ{M}+{M2}")"""

    kind = "ivf_pqr"

    def __init__(self, d, nlist, M, M2, coarse_metric=O.METRIC_L2):
        super().__init__(d, nlist, M, 8, coarse_metric=coarse_metric)
        assert d % M2 == 0
        self.M2, self.dsub2 = int(M2), d // int(M2)
        self.refine_codebooks = None  # [M2, 256, dsub2]
        self.refine_codes = np.zeros((0, self.M2), dtype=np.uint8)
        self.k_factor = 4.0

    def train(self, x):
        super().train(x)
        # the refinement PQ on what PQ1 leaves of the PQ training residuals (the sample of OracleIVFPQ.train)
        x = np.ascontiguousarray(x, dtype=F32)
        maxpts = 256 * self.ksub
        rs = np.random.RandomState(self.train_seed + 1)
        xs = x[rs.permutation(x.shape[0])[:maxpts]] if x.shape[0] > maxpts else x
        la = O.assign(self.coarse_metric, self.centroids, xs)
        r2 = self.residual2(xs, la, super()._encode(xs, la)["codes"])
        cb = np.empty((self.M2, KSUB, self.dsub2), dtype=F32)
        for m2 in range(self.M2):
            cb[m2] = O.kmeans(r2[:, m2 * self.dsub2:(m2 + 1) * self.dsub2], KSUB, self.train_niter,
                              self.train_seed + 2 + self.M + m2)
        self.refine_codebooks = cb

    def residual2(self, x, list_of, codes):
        """r2 = (x - c) - P1[m][code_m], one fp32 rounding per subtraction"""
        r1 = (np.asarray(x, dtype=F32) - self.centroids[np.asarray(list_of, dtype=np.int64)]).astype(F32)
        return (r1 - decode(self.codebooks, codes)).astype(F32)

    def _encode(self, x, list_of):
        rows = super()._encode(x, list_of)
        # the refine codes go by id: _encode sees one add's rows in arrival order
        rc = encode(self.refine_codebooks, self.residual2(x, list_of, rows["codes"]))
        self.refine_codes = np.concatenate([self.refine_codes, rc], axis=0)
        return rows

    def refine(self, x, I1, k):
        """(D, I) [nq, k]: the first-stage candidates I1 [nq, k'] re-ranked on c + PQ1 + PQ2"""
        x = np.ascontiguousarray(x, dtype=F32)
        nq, k1 = I1.shape
        D = np.full((nq, k), O.FLT_MAX, dtype=F32)
        I = np.full((nq, k), -1, dtype=np.int64)
        qi, ji = np.nonzero(I1 >= 0)
        if len(qi) == 0:
            return D, I
        ids = I1[qi, ji]
        inv = np.empty(self.ntotal, dtype=np.int64)
        inv[self.ids] = np.arange(self.ntotal)
        pos = inv[ids]
        r1 = (x[qi] - self.centroids[self.list_of_rows()[pos]]).astype(F32)
        r2 = (r1 - decode(self.codebooks, self.codes[pos])).astype(F32)
        df = (decode(self.refine_codebooks, self.refine_codes[ids]) - r2).astype(F32)
        dis = warp_l2(df)
        for q in range(nq):
            sel = np.nonzero(qi == q)[0]
            order = sel[np.lexsort((ids[sel], dis[sel]))][:k]   # total order (dis asc, id asc)
            D[q, :len(order)] = dis[order]
            I[q, :len(order)] = ids[order]
        return D, I

    def search(self, x, k):
        k1 = first_stage_k(k, self.k_factor)
        if k1 > K_MAX:
            raise RuntimeError(f"k' = {k1} candidates to re-rank, more than {K_MAX}")
        _, I1 = super().search(x, k1)
        return self.refine(x, I1, k)

    def reconstruct_rows(self, ids):
        ids = np.asarray(ids, dtype=np.int64)
        out = super().reconstruct_rows(ids)
        ok = ids >= 0
        out[ok] = (out[ok] + decode(self.refine_codebooks, self.refine_codes[ids[ok]])).astype(F32)
        return out


# ---------------------------------------------------------------- float64 restatement
def reconstruct_f64(state, rows):
    """float64 (c + p1) + p2 of the stored rows `rows` (positions in the list-sorted storage)"""
    list_of = np.repeat(np.arange(state["nlist"]), np.diff(state["list_off"]))[rows]
    ids = np.asarray(state["ids"])[rows]
    cb1 = np.asarray(state["codebooks"], dtype=np.float64)
    cb2 = np.asarray(state["refine_codebooks"], dtype=np.float64)
    return (np.asarray(state["centroids"], dtype=np.float64)[list_of] + decode(cb1, np.asarray(state["codes"])[rows])
            + decode(cb2, np.asarray(state["refine_codes"])[ids]))


# ---------------------------------------------------------------- oracle-backed engine factory
def oracle_engine_factory(cfg):
    """tests/oracle_pq_fs.oracle_engine_factory plus the "IVF{n},PQ{M}+{M2}" factory strings, through the
    parser of distributed_faiss_b200.index.default_engine_factory"""
    from distributed_faiss_b200.index import factory_spec
    from tests.oracle_pq_fs import oracle_engine_factory as others

    spec = factory_spec(cfg)
    if spec is None or spec.kind != "ivf_pqr":
        return others(cfg)
    ix = OracleIVFPQR(cfg.dim, spec.nlist, spec.pq_m, spec.refine_m, coarse_metric=spec.metric)
    if cfg.index_builder_type == "ivf_gpu":
        ix.nprobe = cfg.nprobe
    return ix
