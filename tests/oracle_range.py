"""Range search on the CPU oracles, defined through their k-NN search, which is the accepted truth: a
range search is the oracle's own `search` at k = the most vectors any query can probe (FLAT: ntotal;
IVF: the nprobe longest lists together), cut with faiss's strict comparison (L2: D < radius, inner
product: D > radius) in the float32 the engine compares in.  No distance is restated here.

`oracle_engine_factory` builds the same test doubles as tests/oracle_rflat.oracle_engine_factory with
`range_search` and `search_metric` added, so servers backed by it answer IndexClient.range_search."""
import numpy as np

from oracle import oracle as O

# the kinds whose range search the engine refuses (include/dfx.h, dfx_range_search)
REFUSED = {"ivf_pq_fs": "IVF_PQ_FS (IVF-PQ FastScan)", "ivf_pqr": "IVF_PQR (refined IVF-PQ)"}


def search_metric(ix):
    """the metric of the distances the oracle's search reports: the codecs search in L2"""
    return int(ix.metric) if ix.kind in ("flat", "ivf_flat") else O.METRIC_L2


def probe_bound(ix):
    """at least as many vectors as any query of a search probes"""
    if ix.kind == "flat":
        return int(ix.ntotal)
    lens = np.sort(np.diff(np.asarray(ix.list_off)))[::-1]
    return int(lens[:ix._eff_nprobe()].sum())


def range_search(ix, x, radius):
    """(lims int64[nq + 1], D float32[lims[nq]], I int64[lims[nq]]), each query best first"""
    if ix.kind in REFUSED:
        raise RuntimeError(f"range search is not supported for {REFUSED[ix.kind]} shards")
    if getattr(ix, "refine_flat", 0):
        raise RuntimeError("range search is not supported for shards with a flat refinement (refine_flat)")
    r = np.float32(radius)
    if np.isnan(r):
        raise RuntimeError("range search: the radius is NaN")
    x = np.ascontiguousarray(x, dtype=np.float32)
    D, I = ix.search(x, max(1, probe_bound(ix)))
    keep = (I >= 0) & ((D > r) if search_metric(ix) == O.METRIC_IP else (D < r))
    lims = np.zeros(x.shape[0] + 1, dtype=np.int64)
    np.cumsum(keep.sum(axis=1), out=lims[1:])
    return lims, D[keep], I[keep]


class _RangeMixin:
    @property
    def search_metric(self):
        return search_metric(self)

    def range_search(self, x, radius):
        return range_search(self, x, radius)


_CLASSES = {}


def with_range(ix):
    """the oracle object ix, given `range_search` and `search_metric`"""
    cls = type(ix)
    if cls not in _CLASSES:
        _CLASSES[cls] = type(cls.__name__, (_RangeMixin, cls), {})
    ix.__class__ = _CLASSES[cls]
    return ix


def oracle_engine_factory(cfg):
    from tests.oracle_rflat import oracle_engine_factory as others

    return with_range(others(cfg))
