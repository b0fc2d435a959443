"""faiss `index_factory` strings -> the engine kind that serves them.

The reference lets a deployment describe a shard by a factory string instead of a builder name
("Alternatively, if `index_builder_type` is not specified, one can set `faiss_factory` just like in
FAISS API factory call `faiss.index_factory(...)`", reference README; index.py:385-396), and its
`ivf_gpu` builder takes one too (index.py:71-86).  This module maps the strings that have a kernel
here onto an engine kind.  It is pure: no engine, no torch, so tests use the same parser to build
an oracle-backed engine.

Tokens are case-sensitive, as in faiss:
  "Flat"                          -> flat      (IndexFlat, the given metric)
  "SQfp16"                        -> flat_sq16 (IndexScalarQuantizer QT_fp16, the given metric: every row
                                              stored as its fp16 rounding, 2 d bytes per vector, no
                                              training; searched exactly over the decoded rows)
  "PQ{M}" / "PQ{M}x8"             -> flat_pq   (IndexPQ, 8-bit codes of the raw vectors, the given metric:
                                              M bytes per vector, no lists; M a multiple of 4, at most
                                              128, that divides d)
  "IVF{n},Flat"                   -> ivf_flat  (IndexIVFFlat, the given metric)
  "IVF{n},PQ{M}" / "IVF{n},PQ{M}x8" -> ivf_pq  (IndexIVFPQ, 8-bit codes, L2 only; M a multiple of 4,
                                              at most 128, that divides d)
  "IVF{n},SQfp16"                 -> ivf_sq    (IndexIVFScalarQuantizer QT_fp16, L2 only)
  "IVF{n},SQ8"                    -> ivf_sq8   (IndexIVFScalarQuantizer QT_8bit, L2 only)
  "IVF{n},PQ{M}x4fs"              -> ivf_pq_fs (IndexIVFPQFastScan, 4-bit codes of the raw vectors
                                              (not by_residual), searched through 8-bit quantized
                                              distance tables; L2 only; M a multiple of 8 in
                                              [8, 128] that divides d)
  "IVF{n},PQ{M}+{M2}"             -> ivf_pqr   (IndexIVFPQR: 8-bit IVF-PQ whose residual error is encoded
                                              again by a second 8-bit PQ of M2 bytes; a search re-ranks
                                              the k * k_factor best IVF-PQ candidates on the finer
                                              reconstruction; L2 only; M and M2 each a multiple of 4, at
                                              most 128, that divides d)
  "IVF{n},<codec>,RFlat"          -> the codec's kind with a flat refinement (IndexRefineFlat over the IVF
                                              index): <codec> is PQ{M}, PQ{M}x8, PQ{M}x4fs, SQ8 or SQfp16 with
                                              the limits above; the raw fp32 vectors are kept next to the
                                              lists and a search re-ranks the k * k_factor best candidates
                                              (k_factor 1 by default, as in faiss) on their exact distances;
                                              L2 only
Everything else (OPQ / PCA prefixes, HNSW, IVF{n}_HNSW quantizers, RFlat after Flat, IVF{n},Flat or
PQ{M}+{M2}, every Refine(...) spelling, IDMap, PQ{M}x4, PQ{M}x4fsr, a FastScan block size suffix "_{bbs}",
PQ{M}x4 / PQ{M}x4fs / PQ{M}np / PQ{M} with a suffix without IVF, SQ4 / SQ6, SQ8 or any other scalar quantizer
without IVF (they need trained ranges), SQfp16 with a suffix, malformed n or M) raises RuntimeError.
"""
import re
from typing import NamedTuple

METRIC_INNER_PRODUCT, METRIC_L2 = 0, 1  # faiss enum values

ACCEPTED_FORMS = ("Flat", "SQfp16", "PQ{M}", "PQ{M}x8", "IVF{n},Flat", "IVF{n},PQ{M}", "IVF{n},PQ{M}x8", "IVF{n},PQ{M}x4fs", "IVF{n},PQ{M}+{M2}",
                  "IVF{n},SQfp16", "IVF{n},SQ8", "IVF{n},PQ{M},RFlat", "IVF{n},PQ{M}x8,RFlat", "IVF{n},PQ{M}x4fs,RFlat",
                  "IVF{n},SQfp16,RFlat", "IVF{n},SQ8,RFlat")

_FLAT_PQ = re.compile(r"PQ([1-9][0-9]*)(x8)?")
_IVF = re.compile(r"IVF([1-9][0-9]*),(Flat|PQ([1-9][0-9]*)(x8|x4fs|\+([1-9][0-9]*))?|SQfp16|SQ8)(,RFlat)?")
# one query's fp32 PQ distance table (M x 256 x 4 bytes) must fit in one thread block's shared memory
# (128 KB at M = 128); more would need split or fp16 tables, which are not bit-exact
_PQ_M_MAX = 128


class FactorySpec(NamedTuple):
    """kind: a name of engine.KIND_NAMES ("flat", "flat_sq16", "flat_pq", "ivf_flat", "ivf_pq", "ivf_sq",
    "ivf_sq8", "ivf_pq_fs", "ivf_pqr").  metric: flat / flat_sq16 / flat_pq / ivf_flat: the search metric; the IVF
    codecs: the coarse quantizer's metric (their search is L2).  pq_m: the PQ sub-quantizers (flat_pq and the
    IVF PQ kinds).  refine_m: ivf_pqr's M2 (bytes of the refinement code), else 0.
    refine_flat: the string ends in ",RFlat" (exact re-ranking on stored fp32 vectors)."""
    kind: str
    metric: int
    nlist: int = 0
    pq_m: int = 0
    refine_m: int = 0
    refine_flat: bool = False


def substitute_centroids(factory_string: str, centroids: int) -> str:
    """`{centroids}` -> cfg.centroids, as the reference's factory path does (index.py:391-394);
    a string without the placeholder is used as it is."""
    if "{centroids}" in factory_string:
        return factory_string.format(centroids=int(centroids))
    return factory_string


def parse_factory(dim: int, factory_string: str, metric: int) -> FactorySpec:
    """(dim, factory string, faiss metric) -> FactorySpec, or RuntimeError for a string no kernel
    here serves."""
    s = factory_string if isinstance(factory_string, str) else ""
    if s == "Flat":
        return FactorySpec("flat", int(metric))
    if s == "SQfp16":
        return FactorySpec("flat_sq16", int(metric))
    m = _FLAT_PQ.fullmatch(s)
    if m is not None:
        return FactorySpec("flat_pq", int(metric), 0, _pq_m(factory_string, int(m.group(1)), dim))
    m = _IVF.fullmatch(s)
    # re-ranking an exact index is a no-op, and IVF-PQR has its own refinement: RFlat follows a codec only
    rflat = m is not None and m.group(6) is not None
    if m is None or (rflat and (m.group(2) == "Flat" or m.group(5) is not None)):
        raise RuntimeError(
            f"faiss_factory {factory_string!r} is not supported by the GPU search path; accepted forms: "
            + ", ".join(ACCEPTED_FORMS) + " (n: number of lists, M: PQ sub-quantizers; case-sensitive)")
    nlist, codec = int(m.group(1)), m.group(2)
    if codec == "Flat":
        return FactorySpec("ivf_flat", int(metric), nlist)
    if int(metric) != METRIC_L2:
        raise RuntimeError(
            f"faiss_factory {factory_string!r} with the inner-product metric is not supported: a PQ or SQ "
            "codec searched by inner product needs inner-product distance tables, which no list scan here "
            "has (use metric='l2', or IVF{n},Flat for inner product)")
    if codec.startswith("PQ") and m.group(4) == "x4fs":
        M = int(m.group(3))
        if M % 8 != 0 or M > _PQ_M_MAX or dim % M != 0:
            raise RuntimeError(
                f"faiss_factory {factory_string!r}: the number of FastScan sub-quantizers must be a multiple of 8 "
                f"in [8, {_PQ_M_MAX}] that divides d={dim} (a row of 4-bit codes is whole 32-bit words)")
        return FactorySpec("ivf_pq_fs", int(metric), nlist, M, 0, rflat)
    if codec.startswith("PQ") and m.group(5) is not None:
        M, M2 = int(m.group(3)), int(m.group(5))
        for name, v in (("PQ", M), ("refinement PQ", M2)):
            if v % 4 != 0 or v > _PQ_M_MAX or dim % v != 0:
                raise RuntimeError(
                    f"faiss_factory {factory_string!r}: the number of {name} sub-quantizers must be a multiple of 4, "
                    f"at most {_PQ_M_MAX}, that divides d={dim}, got {v}")
        return FactorySpec("ivf_pqr", int(metric), nlist, M, M2)
    if codec.startswith("PQ"):
        return FactorySpec("ivf_pq", int(metric), nlist, _pq_m(factory_string, int(m.group(3)), dim), 0, rflat)
    return FactorySpec("ivf_sq" if codec == "SQfp16" else "ivf_sq8", int(metric), nlist, 0, 0, rflat)


def _pq_m(factory_string: str, M: int, dim: int) -> int:
    """M of an 8-bit PQ (IVF{n},PQ{M}[x8] and PQ{M}[x8]), or RuntimeError outside the limits"""
    if M % 4 != 0 or M > _PQ_M_MAX or dim % M != 0:
        why = (" (one query's fp32 distance table, M x 256 x 4 bytes, must fit in one thread block's shared "
               "memory)") if M > _PQ_M_MAX else ""
        raise RuntimeError(
            f"faiss_factory {factory_string!r}: the number of PQ sub-quantizers must be a multiple of 4, "
            f"at most {_PQ_M_MAX}, that divides d={dim}{why}")
    return M
