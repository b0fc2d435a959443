"""Restatement of the device build's training (test infrastructure -- NOT product code).

What `dfx_train_impl` (distributed_faiss_b200/csrc/dfx_build.cu, DESIGN.md section 4.6a) trains,
value for value, in numpy float32 on the oracle's assignment.  The stages follow faiss `Clustering`
(Lloyd iterations from a random subset, at most max_points_per_centroid points per centroid, empty
clusters split off a large one) and `ProductQuantizer::train` (one k-means per sub-quantizer on
<= 256 ksub training vectors) [faiss-upstream: restated from knowledge of faiss Clustering.cpp and
ProductQuantizer.cpp, not checked against faiss here]; the random draws and the arithmetic are the
device build's own:

  rng       std::mt19937_64(seed), C++ [rand.eng.mers] with the [rand.predef] parameters
  sample    sample_rows(n, k, seed): perm = 0..n-1; for i < k: j = i + rng() % (n - i),
            swap(perm[i], perm[j]); the rows perm[:k] in that order
  k-means   init = x[sample_rows(n, k, seed)]; every iteration:
              assign  a = oracle.assign(L2, cent, x)  (ties -> the smaller centroid)
              update  per centroid c with rows: s = the fp32 sum of its rows in ascending row
                      order (one rounding per add), cent[c] = s * (1.0f / (float)cnt);
                      a centroid without rows keeps its value
              split   for every empty c, ascending: big = argmax(h) (the first maximum); stop if
                      h[big] < 2; v = cent[big]; even components: cent[c] = v * (1 + 1/1024),
                      cent[big] = v * (1 - 1/1024), odd components the other way round;
                      h[c] = h[big] // 2, h[big] -= h[c]
  train     nt = min(n, mpc * nlist); when nt < n the k-means sample is
            x[sample_rows(n, nt, seed ^ 0x5bd1e995)], else x itself
            coarse centroids = kmeans(sample, nlist, niter, seed)
            PQ kinds: on the first ns = min(nt, 256 ksub) sample rows, the residuals r = x - c under
              the INDEX metric's assignment (IVF-PQ, IVF-PQR) or the raw rows (FastScan, not
              by_residual); codebook m = kmeans(column slice m, ksub, niter, seed + 1 + m)
            IVF-PQR: r2 = r - decode(encode(r)) (tests/oracle_pqr), refinement codebook
              m2 = kmeans(slice m2 of r2, 256, niter, seed + 1 + M + m2)
            IVF-SQ8: on the residuals of the first min(nt, 100000) sample rows,
              [vmin, vmax - vmin] per dimension (tests/oracle_sq8.sq8_train)
            IVF-Flat, IVF-SQ fp16: the coarse centroids only

The oracle's own training (oracle.kmeans, OracleIVFPQ.train) is a different restatement of faiss
(float64 sums, RandomState samples) and is not what the device build computes.
"""
import numpy as np

from oracle import oracle as O
from tests import oracle_pqr as P
from tests import oracle_sq8 as S

F32 = np.float32
MASK64 = (1 << 64) - 1
SUBSAMPLE_SEED_XOR = 0x5bd1e995
SPLIT_EPS = F32(1) / F32(1024)


class MT19937_64:
    """std::mt19937_64"""

    N, MID = 312, 156
    A = 0xB5026F5AA96619E9
    UPPER, LOWER = 0xFFFFFFFF80000000, 0x7FFFFFFF

    def __init__(self, seed):
        mt = [int(seed) & MASK64]
        for i in range(1, self.N):
            mt.append((6364136223846793005 * (mt[-1] ^ (mt[-1] >> 62)) + i) & MASK64)
        self.mt, self.i = mt, self.N

    def _twist(self):
        mt, N, MID, A = self.mt, self.N, self.MID, self.A
        for i in range(N):
            y = (mt[i] & self.UPPER) | (mt[(i + 1) % N] & self.LOWER)
            mt[i] = mt[(i + MID) % N] ^ (y >> 1) ^ (A if y & 1 else 0)
        self.i = 0

    def __call__(self):
        if self.i >= self.N:
            self._twist()
        y = self.mt[self.i]
        self.i += 1
        y ^= (y >> 29) & 0x5555555555555555
        y ^= (y << 17) & 0x71D67FFFEDA60000
        y ^= (y << 37) & 0xFFF7EEE000000000
        y ^= y >> 43
        return y & MASK64


def sample_rows(n, k, seed):
    """the first k entries of a partial Fisher-Yates shuffle of 0..n-1 (gather_random_rows)"""
    rng = MT19937_64(seed)
    perm = np.arange(n, dtype=np.int64)
    for i in range(k):
        j = i + rng() % (n - i)
        perm[i], perm[j] = perm[j], perm[i]
    return perm[:k].copy()


def centroid_update(x, assign, cent):
    """cent[c] = (fp32 sum of c's rows, ascending) * (1.0f / cnt_c); centroids without rows keep
    their value.  Returns (new centroids, counts)."""
    x = np.ascontiguousarray(x, dtype=F32)
    k = cent.shape[0]
    cnt = np.bincount(assign, minlength=k).astype(np.int64)
    order = np.argsort(assign, kind="stable")
    off = np.concatenate([[0], np.cumsum(cnt)])
    s = np.zeros_like(cent, dtype=F32)
    for r in range(int(cnt.max(initial=0))):  # rank r inside every cluster that has r + 1 rows
        live = np.nonzero(cnt > r)[0]
        s[live] = s[live] + x[order[off[live] + r]]
    out = cent.astype(F32, copy=True)
    full = cnt > 0
    inv = F32(1) / cnt[full].astype(F32)
    out[full] = s[full] * inv[:, None]
    return out, cnt


def split_empty(cent, h):
    """split_cluster_kernel over the empty clusters, in place; returns the (empty, big) pairs"""
    d = cent.shape[1]
    up, dn = F32(1) + SPLIT_EPS, F32(1) - SPLIT_EPS
    even = (np.arange(d) % 2) == 0
    splits = []
    for c in range(len(h)):
        if h[c] != 0:
            continue
        big = int(np.argmax(h))
        if h[big] < 2:
            break
        v = cent[big].copy()
        cent[c] = np.where(even, v * up, v * dn)
        cent[big] = np.where(even, v * dn, v * up)
        h[c] = h[big] // 2
        h[big] -= h[c]
        splits.append((c, big))
    return splits


def kmeans(x, k, niter, seed, log=None):
    """kmeans_device.  log (a list) receives, per iteration, a dict of the assignment, the counts
    and the splits."""
    x = np.ascontiguousarray(x, dtype=F32)
    cent = x[sample_rows(x.shape[0], k, seed)].copy()
    for _ in range(niter):
        a = O.assign(O.METRIC_L2, cent, x)
        cent, h = centroid_update(x, a, cent)
        h0 = h.copy()
        splits = split_empty(cent, h)
        if log is not None:
            log.append({"assign": a, "counts": h0, "splits": splits})
    return cent


def _subquantizers(rows, M, ksub, niter, seed0):
    dsub = rows.shape[1] // M
    return np.stack([kmeans(rows[:, m * dsub:(m + 1) * dsub], ksub, niter, seed0 + m) for m in range(M)])


def train(kind, x, nlist, metric=O.METRIC_L2, M=0, nbits=8, M2=0, niter=25, mpc=256, seed=1234, log=None):
    """what the device build trains for `kind` ("ivf_flat", "ivf_sq", "ivf_sq8", "ivf_pq",
    "ivf_pq_fs", "ivf_pqr") from x: a dict of "centroids" and, as the kind needs, "codebooks"
    [M, ksub, dsub], "refine_codebooks" [M2, 256, dsub2], "sq_trained" [2, d].  log receives the
    coarse k-means' iterations (see kmeans)."""
    x = np.ascontiguousarray(x, dtype=F32)
    n = x.shape[0]
    nt = min(n, mpc * nlist)
    xt = x[sample_rows(n, nt, seed ^ SUBSAMPLE_SEED_XOR)] if nt < n else x
    cent = kmeans(xt, nlist, niter, seed, log)
    out = {"centroids": cent}
    if kind in ("ivf_pq", "ivf_pq_fs", "ivf_pqr"):
        ksub = 1 << nbits
        xs = xt[:min(nt, 256 * ksub)]
        rows = xs if kind == "ivf_pq_fs" else xs - cent[O.assign(metric, cent, xs)]
        cb = _subquantizers(rows, M, ksub, niter, seed + 1)
        out["codebooks"] = cb
        if kind == "ivf_pqr":
            r2 = (rows - P.decode(cb, P.encode(cb, rows))).astype(F32)
            out["refine_codebooks"] = _subquantizers(r2, M2, 256, niter, seed + 1 + M)
    elif kind == "ivf_sq8":
        out["sq_trained"] = S.sq8_train(cent, xt[:min(nt, S.TRAIN_ROWS)], metric)
    return out
