"""CPU oracle of the flat refinement (test infrastructure -- NOT product code).

faiss.index_factory(d, "IVF{n},<codec>,RFlat") restated: IndexRefineFlat(base index), k_factor = 1.
The arithmetic is the canonical one of DESIGN.md section 2 [faiss-upstream: restated from knowledge
of faiss IndexRefine.cpp / index_factory.cpp, not checked against faiss here]:

  train   the base kind's training; the refinement store needs none
  add     the base kind's add; the raw fp32 row is stored by id (arrival order), outside the lists
  search  k' = (int64)((float)k * k_factor); the base kind's search for k' candidates, of which only
          the ids are used; for each candidate df = q_i - x_i, acc = fmaf(df, df, acc) in the
          warp-dot order (oracle.warp_dot, mode 1 -- the value an IVF-Flat L2 shard returns for the
          same (q, x)); the k smallest under the total order (dis, id), padded with (FLT_MAX, -1)
  recon   the stored fp32 row

The first stages are the existing oracles: oracle.OracleIVFPQ, tests/oracle_pq_fs, tests/oracle_sq8
and the C oracle's fp16 scalar quantizer (oracle.OracleIVFSQ).
"""
import numpy as np

from oracle import oracle as O
from tests.oracle_pq_fs import OracleIVFPQFastScan
from tests.oracle_pqr import K_MAX, first_stage_k, warp_l2
from tests.oracle_sq8 import OracleIVFSQ8

F32 = np.float32
BASES = {"ivf_pq": O.OracleIVFPQ, "ivf_pq_fs": OracleIVFPQFastScan, "ivf_sq8": OracleIVFSQ8, "ivf_sq": O.OracleIVFSQ}


def refine_exact(x, I1, vecs, k):
    """(D, I) [nq, k]: the candidates I1 [nq, k'] re-ranked on |q - vecs[id]|^2 in the warp-dot order"""
    x = np.ascontiguousarray(x, dtype=F32)
    nq = I1.shape[0]
    D = np.full((nq, k), O.FLT_MAX, dtype=F32)
    I = np.full((nq, k), -1, dtype=np.int64)
    for q in range(nq):
        ids = I1[q][I1[q] >= 0]
        if len(ids) == 0:
            continue
        dis = warp_l2((x[q][None, :] - vecs[ids]).astype(F32))
        order = np.lexsort((ids, dis))[:k]   # total order (dis asc, id asc)
        D[q, :len(order)] = dis[order]
        I[q, :len(order)] = ids[order]
    return D, I


class _RFlat:
    """mixed in before a base oracle class: the refinement store and the re-ranked search"""

    refine_flat = 1   # as the state dict holds it

    def __init__(self, *a, **kw):
        super().__init__(*a, **kw)
        self.refine_vecs = np.zeros((0, self.d), dtype=F32)
        self.k_factor = 1.0   # faiss IndexRefine default

    def add(self, x):
        x = np.ascontiguousarray(x, dtype=F32)
        super().add(x)
        self.refine_vecs = np.concatenate([self.refine_vecs, x], axis=0)

    def search(self, x, k):
        k1 = first_stage_k(k, self.k_factor)
        if k1 > K_MAX:
            raise RuntimeError(f"k' = {k1} candidates to re-rank, more than {K_MAX}")
        _, I1 = super().search(x, k1)
        return refine_exact(x, I1, self.refine_vecs, k)

    def reconstruct_rows(self, ids):
        ids = np.asarray(ids, dtype=np.int64)
        out = np.full((len(ids), self.d), np.nan, dtype=F32)
        ok = ids >= 0
        out[ok] = self.refine_vecs[ids[ok]]
        return out

    def set_param(self, name, value):
        assert name == "k_factor" and 1 <= value <= 16384
        self.k_factor = float(value)

    def set_state(self, st):
        super().set_state(st)
        assert len(self.refine_vecs) == self.ntotal


_CLASSES = {kind: type("RFlat" + base.__name__, (_RFlat, base), {}) for kind, base in BASES.items()}


def make_rflat(kind, d, nlist, M=0, coarse_metric=O.METRIC_L2):
    """the oracle of "IVF{nlist},<codec>,RFlat" for the base kind `kind` (a key of BASES)"""
    cls = _CLASSES[kind]
    if kind == "ivf_pq":
        return cls(d, nlist, M, 8, coarse_metric=coarse_metric)
    if kind == "ivf_pq_fs":
        return cls(d, nlist, M, coarse_metric=coarse_metric)
    return cls(d, nlist, coarse_metric=coarse_metric)


# ---------------------------------------------------------------- float64 cross-check
def exact_f64(xq, vecs, ids):
    """float64 |q - x_id|^2: [nq, len(ids)]"""
    diff = np.asarray(xq, dtype=np.float64)[:, None, :] - np.asarray(vecs, dtype=np.float64)[ids][None, :, :]
    return (diff ** 2).sum(axis=2)


# ---------------------------------------------------------------- oracle-backed engine factory
def oracle_engine_factory(cfg):
    """tests/oracle_pqr.oracle_engine_factory plus the ",RFlat" factory strings, through the parser of
    distributed_faiss_b200.index.default_engine_factory; `k_factor` of the cfg is applied as there"""
    from distributed_faiss_b200.index import factory_spec
    from tests.oracle_pqr import oracle_engine_factory as others

    spec = factory_spec(cfg)
    if spec is None or not spec.refine_flat:
        return others(cfg)
    ix = make_rflat(spec.kind, cfg.dim, spec.nlist, spec.pq_m, coarse_metric=spec.metric)
    if "k_factor" in cfg.extra:
        ix.set_param("k_factor", float(cfg.extra["k_factor"]))
    if cfg.index_builder_type == "ivf_gpu":
        ix.nprobe = cfg.nprobe
    return ix
