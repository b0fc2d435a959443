"""Reader / writer for the faiss on-disk index format, for the four index types the reference's
builders create (reference index.py:94 IndexFlatIP, :36-40 IndexIVFFlat, :43-48 IndexIVFPQ,
:63-68 IndexIVFScalarQuantizer(QT_fp16)), the 8-bit scalar quantizer of the factory string
"IVF{n},SQ8" (IndexIVFScalarQuantizer(QT_8bit)), the fp16 scalar quantizer without lists of the
factory string "SQfp16" (IndexScalarQuantizer(QT_fp16)) and the product quantizer without lists of the
factory string "PQ{M}" (IndexPQ, 8-bit codes); the reference saves shards with
`faiss.write_index(self.faiss_index, index_file)` (index.py:459) and loads them with
`faiss.read_index` (index.py:303).  SURVEY.md section 8(f) next-3.

The engine state dict (engine.GpuIndex.get_state / set_state: centroids, codebooks, list-sorted
codes + shard-local ids + list offsets) maps one-to-one onto what faiss serialises, so a shard
saved by the reference can be loaded straight into HBM and vice versa.  The per-vector IVF-PQ
term `tvals` is not part of the faiss format; the engine recomputes it on import.

STATUS: written from the layout of faiss 1.7.x `impl/index_write.cpp` / `index_read.cpp`; faiss
itself is not available in this environment (SURVEY.md section 8c), so the format is checked for
self-consistency only (tests/test_faiss_io.py), never against a file written by faiss.  The same
holds for the 4-bit IndexIVFPQ codes [faiss-upstream], restated from faiss's PQEncoderGeneric, and for
IndexPQ ("IxPq") [faiss-upstream: index_write.cpp], never compared with a file faiss wrote.
IndexIVFPQFastScan ("IwPf", the factory string "IVF{n},PQ{M}x4fs") is neither read nor written: its
block-interleaved code layout could not be checked without faiss; such shards use the npz format,
with or without a flat refinement.

Layout (little endian, no padding; `vec<T>` = u64 count + raw elements):
  header   : i32 d, i64 ntotal, i64 1<<20, i64 1<<20, u8 is_trained, i32 metric (0 IP, 1 L2)
  flat     : fourcc "IxFI" | "IxF2", header, vec<f32> xb
  SQ       : fourcc "IxSQ", header (with the search metric), SQ (i32 qtype = 4 (fp16), i32 rangestat = 0,
             f32 rangestat_arg = 0, u64 d, u64 code_size = 2 d, vec<f32> trained (empty)), vec<u8> codes
             [ntotal][2 d] (little-endian fp16 of the raw rows, in id order); other qtypes are refused
             [faiss-upstream: IndexScalarQuantizer, index_write.cpp]
  PQ       : fourcc "IxPq", header (with the search metric), PQ (u64 d, u64 M, u64 nbits = 8, vec<f32>
             centroids [M][256][d / M]), vec<u8> codes [ntotal][M] (in id order), i32 search_type = 0
             (ST_PQ: exhaustive ADC), u8 encode_signs = 0, i32 polysemous_ht = 0; other nbits and search
             types are refused [faiss-upstream: IndexPQ, index_write.cpp]
  ivf hdr  : header, u64 nlist, u64 nprobe, <quantizer: flat index of the centroids>,
             u8 direct-map type (0), vec<i64> direct map (empty)
  invlists : fourcc "ilar", u64 nlist, u64 code_size, fourcc "full" + vec<u64> sizes  (or "sprs" +
             vec<u64> (list, size) pairs when at most half of the lists are non-empty), then for
             every non-empty list: codes (size * code_size bytes), ids (size * i64)
  IVFFlat  : "IwFl", ivf hdr, invlists (code = raw f32 vector)
  IVFPQ    : "IwPQ", ivf hdr, u8 by_residual, u64 code_size, PQ (u64 d, u64 M, u64 nbits,
             vec<f32> centroids [M][ksub][dsub]), invlists (code = M bytes; nbits 4: ceil(M / 2)
             bytes, two codes per byte, low nibble first [faiss-upstream: PQEncoderGeneric])
  IVFPQR   : "IwQR", the IVFPQ body (8-bit codes), then the refinement PQ (u64 d, u64 M2, u64 nbits = 8,
             vec<f32> centroids [M2][256][d / M2]), vec<u8> refine codes [ntotal][M2] in id order,
             f32 k_factor [faiss-upstream: IndexIVFPQR, index_write.cpp]
  IVFSQ    : "IwSq", ivf hdr, SQ (i32 qtype, i32 rangestat, f32 rangestat_arg, u64 d,
             u64 code_size, vec<f32> trained), u64 code_size, u8 by_residual, invlists
             qtype 4 (fp16): trained empty, code = d little-endian fp16 of the residual
             qtype 0 (8bit): rangestat 0 (min-max), trained = [vmin (d), vdiff (d)],
                             code = d bytes of the residual
  RefineFlat: "IxRF", header, the base index (IVFPQ with 8-bit codes or IVFSQ, as above), the refine
             index (a flat "IxF2" index holding the raw rows in id order), f32 k_factor
             [faiss-upstream: IndexRefineFlat, index_write.cpp]
"""
import struct
from typing import BinaryIO, Dict, Tuple

import numpy as np

METRIC_IP, METRIC_L2 = 0, 1
QT_8BIT, QT_FP16 = 0, 4


class FaissFormatError(RuntimeError):
    pass


# ------------------------------------------------------------------ primitives
def _w(f: BinaryIO, fmt: str, *vals):
    f.write(struct.pack("<" + fmt, *vals))


def _r(f: BinaryIO, fmt: str):
    size = struct.calcsize("<" + fmt)
    raw = f.read(size)
    if len(raw) != size:
        raise FaissFormatError("unexpected end of file")
    return struct.unpack("<" + fmt, raw)


def _wvec(f: BinaryIO, arr: np.ndarray, dtype):
    arr = np.ascontiguousarray(arr, dtype=dtype).reshape(-1)
    _w(f, "Q", arr.size)
    f.write(arr.tobytes())


def _rvec(f: BinaryIO, dtype) -> np.ndarray:
    (n,) = _r(f, "Q")
    return _rraw(f, n, dtype)


def _rraw(f: BinaryIO, n: int, dtype) -> np.ndarray:
    nbytes = int(n) * np.dtype(dtype).itemsize
    raw = f.read(nbytes)
    if len(raw) != nbytes:
        raise FaissFormatError("unexpected end of file")
    return np.frombuffer(raw, dtype=dtype).copy()


def _fourcc(f: BinaryIO) -> str:
    raw = f.read(4)
    if len(raw) != 4:
        raise FaissFormatError("unexpected end of file")
    return raw.decode("ascii", errors="replace")


def _wheader(f, d, ntotal, metric, is_trained=True):
    _w(f, "iqqqBi", int(d), int(ntotal), 1 << 20, 1 << 20, 1 if is_trained else 0, int(metric))


def _rheader(f):
    d, ntotal, _, _, trained, metric = _r(f, "iqqqBi")
    if metric > 1:
        _r(f, "f")  # metric_arg of the exotic metrics
    return d, ntotal, bool(trained), metric


# ------------------------------------------------------------------ pieces
def _write_flat(f, xb: np.ndarray, metric: int):
    xb = np.ascontiguousarray(xb, dtype=np.float32)
    f.write(b"IxFI" if metric == METRIC_IP else b"IxF2")
    _wheader(f, xb.shape[1], xb.shape[0], metric)
    _wvec(f, xb, np.float32)


def _read_flat_body(f, cc):
    d, ntotal, _, metric = _rheader(f)
    xb = _rvec(f, np.float32)
    if xb.size != d * ntotal:
        raise FaissFormatError(f"flat index: {xb.size} floats for ntotal={ntotal}, d={d}")
    return {"kind": "flat", "d": d, "metric": metric, "xb": xb.reshape(ntotal, d)}


def _write_ivf_header(f, st, metric, coarse_metric, nprobe):
    _wheader(f, st["d"], len(st["ids"]), metric)
    _w(f, "QQ", int(st["nlist"]), int(nprobe))
    _write_flat(f, st["centroids"], coarse_metric)
    _w(f, "B", 0)  # DirectMap::NoMap
    _w(f, "Q", 0)


def _read_ivf_header(f):
    d, ntotal, _, metric = _rheader(f)
    nlist, nprobe = _r(f, "QQ")
    cc = _fourcc(f)
    if cc not in ("IxFI", "IxF2", "IxFl"):
        raise FaissFormatError(f"coarse quantizer {cc!r} is not a flat index")
    q = _read_flat_body(f, cc)
    if q["xb"].shape != (nlist, d):
        raise FaissFormatError("coarse quantizer does not hold nlist centroids")
    (dm_type,) = _r(f, "B")
    _rvec(f, np.int64)
    if dm_type == 2:  # DirectMap::Hashtable: vec of (i64, i64) pairs
        (n,) = _r(f, "Q")
        _rraw(f, 2 * n, np.int64)
    return d, ntotal, metric, nlist, nprobe, q["xb"], q["metric"]


def _write_invlists(f, list_off, ids, rows_u8: np.ndarray, code_size: int):
    list_off = np.asarray(list_off, dtype=np.int64)
    nlist = len(list_off) - 1
    sizes = np.diff(list_off).astype(np.uint64)
    f.write(b"ilar")
    _w(f, "QQ", nlist, int(code_size))
    if int((sizes > 0).sum()) > nlist // 2:
        f.write(b"full")
        _wvec(f, sizes, np.uint64)
    else:
        f.write(b"sprs")
        nz = np.nonzero(sizes)[0]
        _wvec(f, np.stack([nz.astype(np.uint64), sizes[nz]], axis=1), np.uint64)
    ids = np.ascontiguousarray(ids, dtype=np.int64)
    rows_u8 = np.ascontiguousarray(rows_u8).view(np.uint8).reshape(len(ids), code_size)
    for l in range(nlist):
        a, b = int(list_off[l]), int(list_off[l + 1])
        if b > a:
            f.write(rows_u8[a:b].tobytes())
            f.write(ids[a:b].tobytes())


def _read_invlists(f, nlist_expected):
    cc = _fourcc(f)
    if cc == "il00":  # no inverted lists stored
        raise FaissFormatError("index file holds no inverted lists")
    if cc != "ilar":
        raise FaissFormatError(f"inverted lists of type {cc!r} are not supported")
    nlist, code_size = _r(f, "QQ")
    if nlist != nlist_expected:
        raise FaissFormatError("inverted lists / header nlist mismatch")
    lt = _fourcc(f)
    sizes = np.zeros(nlist, dtype=np.int64)
    if lt == "full":
        v = _rvec(f, np.uint64)
        if v.size != nlist:
            raise FaissFormatError("list size table has the wrong length")
        sizes[:] = v
    elif lt == "sprs":
        v = _rvec(f, np.uint64).reshape(-1, 2)
        sizes[v[:, 0].astype(np.int64)] = v[:, 1]
    else:
        raise FaissFormatError(f"unknown list size encoding {lt!r}")
    list_off = np.zeros(nlist + 1, dtype=np.int64)
    np.cumsum(sizes, out=list_off[1:])
    n = int(list_off[-1])
    rows = np.empty((n, code_size), dtype=np.uint8)
    ids = np.empty(n, dtype=np.int64)
    for l in range(nlist):
        a, b = int(list_off[l]), int(list_off[l + 1])
        if b > a:
            rows[a:b] = _rraw(f, (b - a) * code_size, np.uint8).reshape(b - a, code_size)
            ids[a:b] = _rraw(f, b - a, np.int64)
    return list_off, ids, rows, code_size


def _pack_pq_codes(codes: np.ndarray, nbits: int) -> np.ndarray:
    """[n, M] codes, one per byte -> faiss's stored rows.  8 bits: unchanged.  4 bits
    [faiss-upstream: PQEncoderGeneric writes each code's bits least significant first]: code m in the
    low nibble of byte m // 2 when m is even, in the high nibble when odd; an odd M leaves the last
    high nibble 0.  code_size = ceil(M / 2)."""
    if nbits == 8:
        return np.ascontiguousarray(codes, dtype=np.uint8)
    if codes.size and int(codes.max()) >= 16:
        raise FaissFormatError("IndexIVFPQ with 4 bits per sub-quantizer: a code is >= 16")
    n, M = codes.shape
    c = np.zeros((n, M + (M & 1)), dtype=np.uint8)
    c[:, :M] = codes
    return np.ascontiguousarray(c[:, 0::2] | (c[:, 1::2] << 4))


def _unpack_pq_codes(rows: np.ndarray, M: int, nbits: int) -> np.ndarray:
    """faiss's stored rows -> [n, M] codes, one per byte (the inverse of _pack_pq_codes)"""
    if nbits == 8:
        return rows.reshape(-1, M)
    out = np.empty((rows.shape[0], 2 * rows.shape[1]), dtype=np.uint8)
    out[:, 0::2] = rows & 15
    out[:, 1::2] = rows >> 4
    return np.ascontiguousarray(out[:, :M])


# ------------------------------------------------------------------ public
def write_index(state: Dict, path: str, nprobe: int = 1) -> None:
    """state: engine / oracle `get_state()` dict.  Writes a faiss index file."""
    kind = state["kind"]
    with open(path, "wb") as f:
        if state.get("refine_flat"):
            # IndexRefineFlat around the base index; the base's own refusals (FastScan) apply below
            if kind not in ("ivf_pq", "ivf_pq_fs", "ivf_sq", "ivf_sq8") or (kind == "ivf_pq" and int(state["ksub"]) != 256):
                raise FaissFormatError(f"IndexRefineFlat over an index of kind {kind!r} is not served")
            vecs = np.ascontiguousarray(state["refine_vecs"], dtype=np.float32).reshape(-1, int(state["d"]))
            if len(vecs) != len(state["ids"]):
                raise FaissFormatError("IndexRefineFlat: the refine index does not hold ntotal vectors")
            if kind != "ivf_pq_fs":
                f.write(b"IxRF")
                _wheader(f, state["d"], len(state["ids"]), METRIC_L2)
        if kind == "flat":
            _write_flat(f, state["xb"], int(state["metric"]))
        elif kind == "flat_sq16":
            d = int(state["d"])
            c16 = np.ascontiguousarray(state["codes16"], dtype="<u2").reshape(-1, d)
            f.write(b"IxSQ")
            _wheader(f, d, c16.shape[0], int(state["metric"]))
            _w(f, "iif", QT_FP16, 0, 0.0)
            _w(f, "QQ", d, 2 * d)
            _w(f, "Q", 0)  # trained: empty for fp16
            _wvec(f, c16.view(np.uint8), np.uint8)
        elif kind == "flat_pq":
            d, M = int(state["d"]), int(state["M"])
            if int(state["ksub"]) != 256:
                raise FaissFormatError(f"IndexPQ: 8-bit codes only, got ksub={int(state['ksub'])}")
            codes = np.ascontiguousarray(state["codes"], dtype=np.uint8).reshape(-1, M)
            f.write(b"IxPq")
            _wheader(f, d, codes.shape[0], int(state["metric"]))
            _w(f, "QQQ", d, M, 8)
            _wvec(f, state["codebooks"], np.float32)
            _wvec(f, codes, np.uint8)
            _w(f, "iBi", 0, 0, 0)  # search_type ST_PQ, encode_signs, polysemous_ht
        elif kind == "ivf_flat":
            f.write(b"IwFl")
            _write_ivf_header(f, state, int(state["metric"]), int(state["metric"]), nprobe)
            vecs = np.ascontiguousarray(state["vecs"], dtype=np.float32)
            _write_invlists(f, state["list_off"], state["ids"], vecs, 4 * int(state["d"]))
        elif kind in ("ivf_pq", "ivf_pqr"):
            M, ksub = int(state["M"]), int(state["ksub"])
            nbits = {256: 8, 16: 4}.get(ksub)
            if nbits is None:
                raise FaissFormatError(f"only 8-bit and 4-bit product quantizers are supported, got ksub={ksub}")
            codes = _pack_pq_codes(np.asarray(state["codes"], dtype=np.uint8).reshape(-1, M), nbits)
            if kind == "ivf_pqr" and nbits != 8:
                raise FaissFormatError(f"IndexIVFPQR: 8-bit codes only, got ksub={ksub}")
            f.write(b"IwPQ" if kind == "ivf_pq" else b"IwQR")
            _write_ivf_header(f, state, METRIC_L2, int(state["coarse_metric"]), nprobe)
            _w(f, "B", 1)  # by_residual
            _w(f, "Q", codes.shape[1])  # code_size
            _w(f, "QQQ", int(state["d"]), M, nbits)
            _wvec(f, state["codebooks"], np.float32)
            _write_invlists(f, state["list_off"], state["ids"], codes, codes.shape[1])
            if kind == "ivf_pqr":
                M2 = int(state["M2"])
                _w(f, "QQQ", int(state["d"]), M2, 8)
                _wvec(f, state["refine_codebooks"], np.float32)
                _wvec(f, np.asarray(state["refine_codes"], dtype=np.uint8).reshape(-1, M2), np.uint8)
                _w(f, "f", float(state.get("k_factor", 4.0)))
        elif kind == "ivf_pq_fs":
            # faiss stores FastScan codes (IwPf) in blocks of bbs vectors with the nibbles permuted for
            # its SIMD lookups; that layout has never been checked against faiss, so it is not written
            raise FaissFormatError("IndexIVFPQFastScan (IVF{n},PQ{M}x4fs) shards cannot be written in the faiss "
                                   "format; save them with the default npz format (index_format='dfx')")
        elif kind == "ivf_sq":
            d = int(state["d"])
            f.write(b"IwSq")
            _write_ivf_header(f, state, METRIC_L2, int(state["coarse_metric"]), nprobe)
            _w(f, "iif", QT_FP16, 0, 0.0)
            _w(f, "QQ", d, 2 * d)
            _w(f, "Q", 0)  # trained: empty for fp16
            _w(f, "Q", 2 * d)
            _w(f, "B", 1)  # by_residual
            c16 = np.ascontiguousarray(state["codes16"], dtype="<u2")
            _write_invlists(f, state["list_off"], state["ids"], c16, 2 * d)
        elif kind == "ivf_sq8":
            d = int(state["d"])
            f.write(b"IwSq")
            _write_ivf_header(f, state, METRIC_L2, int(state["coarse_metric"]), nprobe)
            _w(f, "iif", QT_8BIT, 0, 0.0)  # rangestat 0 = RS_minmax, rangestat_arg 0
            _w(f, "QQ", d, d)
            _wvec(f, np.asarray(state["sq_trained"], dtype=np.float32).reshape(2 * d), np.float32)
            _w(f, "Q", d)
            _w(f, "B", 1)  # by_residual
            _write_invlists(f, state["list_off"], state["ids"], np.ascontiguousarray(state["codes8"], np.uint8), d)
        else:
            raise FaissFormatError(f"unknown index kind {kind!r}")
        if state.get("refine_flat"):
            _write_flat(f, vecs, METRIC_L2)
            _w(f, "f", float(state.get("k_factor", 1.0)))


def read_index(path: str) -> Tuple[Dict, int]:
    """Returns (state dict for `set_state`, nprobe stored in the file)."""
    with open(path, "rb") as f:
        cc = _fourcc(f)
        if cc == "IxRF":
            d, ntotal, _, metric = _rheader(f)
            st, nprobe = _read_one(f, _fourcc(f))
            four_bit = st["kind"] == "ivf_pq" and st["ksub"] != 256
            if st["kind"] not in ("ivf_pq", "ivf_sq", "ivf_sq8") or four_bit or metric != METRIC_L2:
                raise FaissFormatError(f"IndexRefineFlat over an index of kind {st['kind']!r}"
                                       f"{' with 4-bit codes' if four_bit else ''} (metric {metric}) is not served")
            rcc = _fourcc(f)
            if rcc not in ("IxF2", "IxFl"):
                raise FaissFormatError(f"IndexRefineFlat: the refine index {rcc!r} is not a flat L2 index")
            flat = _read_flat_body(f, rcc)
            (k_factor,) = _r(f, "f")
            if flat["d"] != d or st["d"] != d or flat["xb"].shape[0] != ntotal or len(st["ids"]) != ntotal:
                raise FaissFormatError("IndexRefineFlat: the refine index does not hold the base index's vectors")
            st.update(refine_flat=1, refine_vecs=flat["xb"], k_factor=float(k_factor))
            return st, nprobe
        return _read_one(f, cc)


def _read_one(f: BinaryIO, cc: str) -> Tuple[Dict, int]:
    """one index whose fourcc `cc` has been read"""
    if cc in ("IxFI", "IxF2", "IxFl"):
        st = _read_flat_body(f, cc)
        return st, 1
    if cc == "IxSQ":
        d, ntotal, _, metric = _rheader(f)
        qtype, _, _ = _r(f, "iif")
        sd, scs = _r(f, "QQ")
        trained = _rvec(f, np.float32)
        codes = _rvec(f, np.uint8)
        if qtype != QT_FP16 or sd != d or scs != 2 * d or trained.size != 0:
            raise FaissFormatError(f"IndexScalarQuantizer: only QT_fp16 (qtype {QT_FP16}) with 2 * d bytes per "
                                   f"vector is supported (qtype={qtype}, d={sd}, code_size={scs})")
        if metric not in (METRIC_IP, METRIC_L2):
            raise FaissFormatError(f"IndexScalarQuantizer: metric {metric} is not supported")
        if codes.size != ntotal * 2 * d:
            raise FaissFormatError("IndexScalarQuantizer: the codes do not hold ntotal vectors")
        return {"kind": "flat_sq16", "d": d, "metric": metric, "codes16": codes.view("<u2").reshape(ntotal, d)}, 1
    if cc == "IxPq":
        d, ntotal, _, metric = _rheader(f)
        pd, M, nbits = _r(f, "QQQ")
        cb = _rvec(f, np.float32)
        codes = _rvec(f, np.uint8)
        search_type, _, _ = _r(f, "iBi")
        if nbits != 8 or pd != d or M == 0 or d % M != 0 or cb.size != M * 256 * (d // M):
            raise FaissFormatError(f"IndexPQ: only 8 bits per sub-quantizer with M dividing d is supported "
                                   f"(nbits={nbits}, M={M}, d={pd})")
        if search_type != 0:
            raise FaissFormatError(f"IndexPQ: only search_type 0 (ST_PQ, exhaustive ADC) is supported, got {search_type}")
        if metric not in (METRIC_IP, METRIC_L2):
            raise FaissFormatError(f"IndexPQ: metric {metric} is not supported")
        if codes.size != ntotal * M:
            raise FaissFormatError("IndexPQ: the codes do not hold ntotal vectors")
        return {"kind": "flat_pq", "d": d, "metric": metric, "M": int(M), "ksub": 256,
                "codebooks": cb.reshape(M, 256, d // M), "codes": codes.reshape(ntotal, M)}, 1
    if cc not in ("IwFl", "IwPQ", "IwQR", "IwSq"):
        raise FaissFormatError(
            f"faiss index type {cc!r} is not one of the types the GPU search path serves "
            "(IndexFlat, IndexScalarQuantizer fp16, IndexPQ, IndexIVFFlat, IndexIVFPQ, IndexIVFPQR, "
            "IndexIVFScalarQuantizer fp16 / 8bit)")
    d, ntotal, metric, nlist, nprobe, cent, cmetric = _read_ivf_header(f)
    st = {"d": d, "nlist": nlist, "centroids": cent}
    if cc == "IwFl":
        list_off, ids, rows, cs = _read_invlists(f, nlist)
        if cs != 4 * d:
            raise FaissFormatError("IndexIVFFlat code size is not 4 * d")
        st.update(kind="ivf_flat", metric=metric, vecs=rows.view(np.float32).reshape(-1, d))
    elif cc in ("IwPQ", "IwQR"):
        (by_res,) = _r(f, "B")
        (code_size,) = _r(f, "Q")
        pd, M, nbits = _r(f, "QQQ")
        cb = _rvec(f, np.float32)
        if not by_res or nbits not in (8, 4) or pd != d or code_size != (M * nbits + 7) // 8:
            raise FaissFormatError("IndexIVFPQ: only by_residual with 8 or 4 bits per sub-quantizer is "
                                   f"supported (nbits={nbits}, M={M}, code_size={code_size})")
        if metric != METRIC_L2:
            raise FaissFormatError("IndexIVFPQ: only METRIC_L2 is supported")
        list_off, ids, rows, cs = _read_invlists(f, nlist)
        if cs != code_size:
            raise FaissFormatError("IndexIVFPQ: inverted lists / header code_size mismatch")
        ksub = 1 << nbits
        st.update(kind="ivf_pq", coarse_metric=cmetric, M=M, ksub=ksub,
                  codebooks=cb.reshape(M, ksub, d // M), codes=_unpack_pq_codes(rows, M, nbits))
        if cc == "IwQR":
            rd, M2, nbits2 = _r(f, "QQQ")
            rcb = _rvec(f, np.float32)
            rcodes = _rvec(f, np.uint8)
            (k_factor,) = _r(f, "f")
            if nbits != 8 or nbits2 != 8 or rd != d or M2 == 0 or d % M2 != 0 or rcb.size != M2 * 256 * (d // M2):
                raise FaissFormatError(f"IndexIVFPQR: only 8-bit codes in both product quantizers are supported "
                                       f"(nbits={nbits}, refine nbits={nbits2}, M2={M2}, d={d})")
            if rcodes.size != ntotal * M2:
                raise FaissFormatError("IndexIVFPQR: the refine codes do not hold ntotal vectors")
            st.update(kind="ivf_pqr", M2=int(M2), refine_codebooks=rcb.reshape(M2, 256, d // M2),
                      refine_codes=rcodes.reshape(ntotal, M2), k_factor=float(k_factor))
    else:
        qtype, rangestat, _ = _r(f, "iif")
        sd, scs = _r(f, "QQ")
        trained = _rvec(f, np.float32)
        (code_size,) = _r(f, "Q")
        (by_res,) = _r(f, "B")
        if qtype == QT_8BIT:
            if not by_res or code_size != d or trained.size != 2 * d:
                raise FaissFormatError("IndexIVFScalarQuantizer QT_8bit: only by_residual with d codes "
                                       "and a [vmin, vdiff] trained vector is supported")
            list_off, ids, rows, cs = _read_invlists(f, nlist)
            st.update(kind="ivf_sq8", coarse_metric=cmetric, sq_trained=trained.reshape(2, d),
                      codes8=rows.reshape(-1, d))
        else:
            if qtype != QT_FP16 or not by_res or code_size != 2 * d:
                raise FaissFormatError("IndexIVFScalarQuantizer: only QT_fp16 and QT_8bit, by_residual, "
                                       "are supported")
            list_off, ids, rows, cs = _read_invlists(f, nlist)
            st.update(kind="ivf_sq", coarse_metric=cmetric, codes16=rows.view("<u2").reshape(-1, d))
    if len(ids) != ntotal:
        raise FaissFormatError("inverted lists do not hold ntotal vectors")
    st.update(list_off=list_off, ids=ids)
    return st, int(nprobe)
