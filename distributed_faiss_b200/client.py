"""IndexClient: fan a query out to every shard and merge the per-shard top-k.

API mirror of the reference's `IndexClient` (distributed_faiss/client.py:57-345): same
constructor (discovery file `N\\nhost,port\\n...`, client.py:87-120), same method names,
same round-robin placement of added batches (client.py:186-192), same return contract of
`search` -- `(float32[nq,k] ascending, list[nq][k] of metadata)`, scores NEGATED for
metric "dot" (client.py:291-292), shards that returned fewer than k hits padded out.

What is different underneath: the k-way merge that the reference runs on the CPU with
faiss's `float_maxheap_array_t` (client.py:29-54) is the CUDA merge kernel K6 of libdfx
(same semantics, pinned by the reference's golden vectors), and when the client's process
hosts a `spmd.SearchPlane` (one process per GPU under torchrun, the client in the process of
plane rank 0) `search` / `search_with_filter` run as ONE collective: query broadcast,
per-shard search, one all-gather of the packed (D, I) blocks and the merge all stay on the
GPUs and travel over NCCL/NVLink; the pickled sockets (rpc.py) remain for the control plane
and for the metadata OBJECTS of the winners.  Without a plane every call uses the sockets,
exactly like the reference.
"""
import collections.abc
import itertools
import logging
import os
import random
import time
from multiprocessing.dummy import Pool as ThreadPool
from typing import Callable, List, Optional, Tuple

import numpy as np

from . import rpc
from .index_cfg import IndexCfg
from .index_state import IndexState

logger = logging.getLogger("distributed_faiss_b200")


def _device_merge(Dall: np.ndarray, Iall: np.ndarray, negate: bool):
    from . import engine

    return engine.merge(Dall, Iall, negate=negate)


class MetaRows(collections.abc.Sequence):
    """`list[nq]` of `list[k]` of integer metadata, backed by the int64 matrix the device
    returned (negative = no result -> None).  Behaves like the reference's list of lists
    (indexing, iteration, len, == with lists); `tolist()` materialises it.  Building 40 960 Python
    ints eagerly would cost more than the whole 8-GPU search of a 4096-query batch."""

    __slots__ = ("_a",)

    def __init__(self, a: np.ndarray):
        self._a = a

    def __len__(self):
        return self._a.shape[0]

    def _row(self, r):
        row = r.tolist()
        return [v if v >= 0 else None for v in row] if (r < 0).any() else row

    def __getitem__(self, i):
        if isinstance(i, slice):
            return [self._row(r) for r in self._a[i]]
        return self._row(self._a[i])

    def __iter__(self):
        return (self._row(r) for r in self._a)

    def __eq__(self, other):
        if isinstance(other, MetaRows):
            return np.array_equal(self._a, other._a)
        try:
            return self.tolist() == list(other)
        except TypeError:
            return NotImplemented

    def __ne__(self, other):
        r = self.__eq__(other)
        return r if r is NotImplemented else not r

    def __repr__(self):
        return repr(self.tolist())

    def tolist(self):
        return [self._row(r) for r in self._a]

    @property
    def array(self) -> np.ndarray:
        return self._a


class ResultHeap:
    """Accumulates per-shard (D, I) blocks and merges them on `finalize` (client.py:29-54).
    The reference pushes block by block into a faiss heap; here the blocks are stacked and
    merged by one launch of the device merge kernel -- same result, same tie rule (earlier
    block wins among equal values)."""

    merge_backend: Callable = staticmethod(_device_merge)

    def __init__(self, nq, k):
        self.nq, self.k = nq, k
        self.I = np.full((nq, k), -1, dtype="int64")
        self.D = np.full((nq, k), np.finfo(np.float32).max, dtype="float32")
        self._D, self._I = [], []

    def add_result(self, D, I):
        assert D.shape == (self.nq, self.k) and I.shape == (self.nq, self.k)
        self._D.append(np.ascontiguousarray(D, dtype=np.float32))
        self._I.append(np.ascontiguousarray(I, dtype=np.int64))

    def finalize(self):
        if self._D:
            self.D, self.I = type(self).merge_backend(np.stack(self._D), np.stack(self._I), False)


class IndexClient:
    def __init__(self, server_list_path: str, cfg_path: Optional[str] = None):
        machine_ports = IndexClient.read_server_list(server_list_path)
        self.sub_indexes = IndexClient.setup_connection(machine_ports)
        self.num_indexes = len(self.sub_indexes)
        ranks = [s.get_rank() for s in self.sub_indexes]
        self.index_rank_to_id = {rank: pos for pos, rank in enumerate(ranks)}
        self.pool = ThreadPool(self.num_indexes)  # one thread per shard connection
        self.verbose = False
        self.cur_server_ids = {}
        random.seed(time.time())
        self.cfg = IndexCfg.from_json(cfg_path) if cfg_path is not None else None
        # NCCL data plane: attached when this process hosts a spmd.SearchPlane covering exactly
        # the servers of the discovery file (rank-major); None = every call goes over the sockets
        self.plane = None
        self._meta_kind = {}      # index_id -> "int" | "object" (asked over the control plane)
        self.lazy_metadata = True  # int fast path returns MetaRows instead of eager lists
        self._attach_plane()

    # ------------------------------------------------------------ discovery / connections
    @staticmethod
    def read_server_list(server_list_path, initial_timeout=0.1, backoff_factor=1.5,
                         total_max_timeout=7200) -> List[Tuple[str, int]]:
        """File format: first line = expected number of servers, then one `host,port` per
        line.  Polls with exponential back-off until all servers have registered."""
        waited, pause = 0.0, initial_timeout
        while True:
            with open(server_list_path) as fh:
                lines = fh.read().splitlines()
            expected = int(lines[0])
            servers = [(ln.split(",")[0], int(ln.split(",")[1])) for ln in lines[1:] if ln.strip()]
            msg = f"{expected} != {len(servers)} in server list {server_list_path}."
            if expected == len(servers):
                return servers
            print(msg + f" Waiting {round(pause * 100) / 100} seconds for servers to load...")
            time.sleep(pause)
            if waited + pause >= total_max_timeout:
                raise AssertionError(msg + f" Timed out after waiting {round(waited * 100) / 100} seconds")
            waited += pause
            pause *= backoff_factor

    @staticmethod
    def setup_connection(machine_ports) -> List[rpc.Client]:
        return [rpc.Client(i, host, port, False) for i, (host, port) in enumerate(machine_ports)]

    def _all(self, fn):
        return self.pool.map(fn, self.sub_indexes)

    def _attach_plane(self, plane=None):
        from . import spmd

        plane = plane or spmd.current_plane()
        if plane is None or plane.rank != 0 or plane.num_servers != self.num_indexes:
            return False
        if sorted(self.index_rank_to_id) != list(range(self.num_indexes)):
            return False
        self.plane = plane
        return True

    def detach_plane(self):
        self.plane = None

    # ------------------------------------------------------------ control plane
    def create_index(self, index_id: str, cfg: Optional[IndexCfg] = None):
        self._meta_kind.pop(index_id, None)
        if cfg is not None:
            self.cfg = cfg
        if self.cfg is None:
            self.cfg = IndexCfg()
        return self._all(lambda s: s.create_index(index_id, self.cfg))

    def drop_index(self, index_id: str):
        self._all(lambda s: s.drop_index(index_id))

    def save_index(self, index_id: str):
        self._all(lambda s: s.save_index(index_id))

    def load_index(self, index_id: str, cfg: Optional[IndexCfg] = None, force_reload: bool = True) -> bool:
        self._meta_kind.pop(index_id, None)
        if force_reload:
            self._all(lambda s: s.drop_index(index_id))
        loaded = self._all(lambda s: s.load_index(index_id, cfg))
        if cfg is None:
            paths = self._all(lambda s: s.get_config_path(index_id))
            cfg = IndexCfg.from_json(paths[0]) if paths and os.path.isfile(paths[0]) else IndexCfg()
        self.cfg = cfg
        if all(loaded):
            return True
        if any(loaded):
            logger.warning("Some server nodes can't load index: %s", loaded)
        return False

    def add_index_data(self, index_id: str, embeddings: np.ndarray, metadata: Optional[List[object]] = None,
                       train_async_if_triggered: bool = True) -> None:
        """First batch of an index goes to a random shard, then round-robin (client.py:186-192)."""
        self._meta_kind.pop(index_id, None)
        if index_id not in self.cur_server_ids:
            self.cur_server_ids[index_id] = random.randint(0, self.num_indexes - 1)
        target = self.cur_server_ids[index_id]
        self.sub_indexes[target].add_index_data(index_id, embeddings, metadata, train_async_if_triggered)
        self.cur_server_ids[index_id] = (target + 1) % self.num_indexes

    def sync_train(self, index_id: str) -> None:
        self._all(lambda s: s.sync_train(index_id))

    def async_train(self, index_id: str):
        self._all(lambda s: s.sync_train(index_id))

    def add_buffer_to_index(self, index_id: str):
        self._all(lambda s: s.add_buffer_to_index(index_id))

    def get_centroids(self, index_id: str):
        return self._all(lambda s: s.get_centroids(index_id))

    def set_nprobe(self, index_id: str, nprobe: int):
        return self._all(lambda s: s.set_nprobe(index_id, nprobe))

    def get_state(self, index_id: str) -> IndexState:
        return IndexState.get_aggregated_states(self._all(lambda s: s.get_state(index_id)))

    def get_ntotal(self, index_id: str) -> int:
        return sum(self._all(lambda s: s.get_ntotal(index_id)))

    def get_ids(self, index_id: str) -> set:
        return set().union(*self._all(lambda s: s.get_ids(index_id)))

    def set_omp_num_threads(self, num_threads: int) -> None:
        # no server implements it in the reference either (SURVEY.md A.8): raises ServerException
        self._all(lambda s: s.set_omp_num_threads(num_threads))

    def get_num_servers(self):
        return self.num_indexes

    def close(self):
        for conn in self.sub_indexes:
            conn.close()

    # ------------------------------------------------------------ the hot path
    MAX_TOPK = 4096   # per-query results the engine selects, for every index kind; DESIGN.md §7

    def _check_topk(self, topk: int):
        """the reference passes any k to faiss; here the limit is the engine's -- say so on the
        client instead of surfacing it as a ServerException from every shard"""
        if not 1 <= int(topk) <= self.MAX_TOPK:
            raise ValueError(f"topk={topk}: this engine returns 1..{self.MAX_TOPK} results per query; "
                             "search_with_filter over-fetches 3x")

    def search(self, query, topk: int, index_id: str, return_embeddings: bool = False) -> Tuple[np.ndarray, List]:
        self._check_topk(topk)
        maximize_metric: bool = self.cfg.metric == "dot"
        if self.plane is not None:
            return self._search_plane(query, topk, index_id, return_embeddings, maximize_metric)
        results = self.pool.imap(lambda s: s.search(index_id, query, topk, return_embeddings), self.sub_indexes)
        return self._aggregate_results(results, topk, query.shape[0], maximize_metric, return_embeddings)

    def search_with_filter(self, query: np.ndarray, top_k: int, index_id: str, filter_pos: int = -1,
                           filter_value=None) -> Tuple[np.ndarray, List[List[object]]]:
        """Over-fetch 3x and drop results whose metadata[filter_pos] == filter_value
        (client.py:213-263).  Returns per-query lists (possibly shorter than top_k)."""
        if filter_pos < 0:
            return self.search(query, top_k, index_id)
        self._check_topk(3 * top_k)
        if self.plane is not None:
            return self._search_with_filter_plane(query, top_k, index_id, filter_pos, filter_value)
        scores, meta = self.search(query, 3 * top_k, index_id)
        out_scores, out_meta = [], []
        for row_scores, row_meta in zip(scores, meta):
            kept = [(s, m) for s, m in zip(row_scores, row_meta)
                    if m and len(m) > filter_pos and m[filter_pos] != filter_value][:top_k]
            out_meta.append([m for _, m in kept])
            out_scores.append(np.array([s for s, _ in kept], dtype=np.float32).reshape(-1, 1))
        return out_scores, out_meta

    def range_search(self, query: np.ndarray, radius: float, index_id: str, return_embeddings: bool = False
                     ) -> Tuple:
        """Every indexed vector within `radius` of each query, faiss's `range_search` over all shards:
        `(lims int64[nq + 1], scores float32[lims[-1]], meta)`, query i's results at lims[i]:lims[i + 1]
        and `meta` a flat list of their metadata.  A shard keeps what its `search` would score with a
        distance strictly inside the radius: L2 distance < radius, or inner product > radius, by the
        shard's search metric (a `flat` index is always inner product; the codecs search in L2 whatever
        `metric` says).  Each query's results are merged best first; among equal scores the earlier
        shard, then the shard's own order, comes first.  The scores are faiss's values: unlike
        `search`, which negates them for metric "dot" as the reference does, they are never negated.
        With `return_embeddings` a fourth item `embs` float32[lims[-1], d] holds the hits' vectors in
        result order, decoded by their shards (the stored fp32 row of a `,RFlat` shard).
        Over the search plane when one is attached (one collective; the merge runs on the GPU and a
        call returns at most 2^27 hits over all shards), else over the sockets; both return the same."""
        if self.plane is not None:
            return self._range_search_plane(query, radius, index_id, return_embeddings)
        results = self._all(lambda s: s.range_search(index_id, query, radius, return_embeddings))
        metrics = {int(r[3]) for r in results}
        if len(metrics) > 1:
            raise RuntimeError(self._range_metrics_differ(index_id, metrics))
        maximize = metrics == {0}  # faiss METRIC_INNER_PRODUCT
        nq = int(np.asarray(query).shape[0])
        qs, scores, meta = [], [], []
        for lims, D, m, *_ in results:
            qs.append(np.repeat(np.arange(nq, dtype=np.int64), np.diff(lims)))
            scores.append(np.asarray(D, dtype=np.float32))
            meta.extend(m)
        q = np.concatenate(qs)
        D = np.concatenate(scores)
        # the concatenation is shard-major and each shard's segment is sorted, so a stable sort by
        # (query, score) keeps shard order and then the shard's order among equal scores
        order = np.lexsort((-D if maximize else D, q))
        lims = np.zeros(nq + 1, dtype=np.int64)
        np.cumsum(np.bincount(q, minlength=nq), out=lims[1:])
        out = (lims, D[order], [meta[i] for i in order.tolist()])
        if not return_embeddings:
            return out
        d = int(np.asarray(query).shape[1])
        embs = np.concatenate([np.asarray(r[4], dtype=np.float32).reshape(-1, d) for r in results])
        return out + (embs[order],)

    @staticmethod
    def _range_metrics_differ(index_id, metrics):
        return (f"range_search: the shards of index {index_id!r} report different search metrics "
                f"{sorted(metrics)}; their distances cannot be merged")

    # ---- NCCL data plane (spmd.SearchPlane): same contracts, one collective instead of S RPCs
    def _get_meta_kind(self, index_id: str) -> str:
        kind = self._meta_kind.get(index_id)
        if kind is None:
            kinds = self._all(lambda s: s.get_meta_kind(index_id))
            kind = "int" if all(k == "int" for k in kinds) else "object"
            self._meta_kind[index_id] = kind
        return kind

    def _exchange_ids_to_meta(self, index_id: str, I: np.ndarray) -> List[List[object]]:
        """exchange ids ((server rank << 40) | local id) -> metadata objects: shards hosted by this
        process are read directly, the others over their control-plane socket"""
        from . import spmd

        flat = I.reshape(-1)
        out = np.empty(flat.shape[0], dtype=object)  # None where I < 0
        valid = flat >= 0
        owner = np.where(valid, (flat >> spmd.LOCAL_BITS) & 0xFFFFF, -1)
        local = flat & spmd.LOCAL_MASK
        for sr in np.unique(owner[valid]).tolist():
            sel = np.nonzero(owner == sr)[0]
            srv = self.plane.owner_of(int(sr))
            if srv is not None:
                metas = srv.lookup_meta(index_id, local[sel])
            else:
                metas = self.sub_indexes[self.index_rank_to_id[int(sr)]].lookup_meta(index_id, local[sel])
            tmp = np.empty(len(metas), dtype=object)
            tmp[:] = metas
            out[sel] = tmp
        return out.reshape(I.shape).tolist()

    def _search_plane(self, query, topk, index_id, return_embeddings, maximize_metric):
        from . import spmd

        for attempt in (0, 1):
            int_meta = self._get_meta_kind(index_id) == "int"
            try:
                D, I, _cnt, embs, meta_int = self.plane.search(
                    index_id, query, topk, maximize=maximize_metric, return_embeddings=return_embeddings,
                    int_meta=int_meta)
                break
            except spmd.MetaKindChanged:
                self._meta_kind.pop(index_id, None)
                if attempt:
                    raise
            except spmd.PlaneError as e:
                raise rpc.ServerException(str(e))
        if int_meta:
            # with embeddings I holds exchange ids (the owners decoded by them) and the integer
            # metadata of the winners came back separately
            ids = np.where(I < 0, -1, meta_int) if return_embeddings else I
            meta = MetaRows(ids) if self.lazy_metadata else MetaRows(ids).tolist()
        else:
            meta = self._exchange_ids_to_meta(index_id, I)
        if not return_embeddings:
            return D, meta
        # the reference returns list[nq][k] of per-winner vectors (client.py:299-307)
        picked = [[embs[q, j] if I[q, j] >= 0 else None for j in range(I.shape[1])] for q in range(I.shape[0])]
        return D, meta, picked

    def _range_search_plane(self, query, radius, index_id, return_embeddings):
        from . import spmd

        for attempt in (0, 1):
            int_meta = self._get_meta_kind(index_id) == "int"
            try:
                lims, D, P, embs = self.plane.range_search(index_id, query, radius, int_meta=int_meta,
                                                           return_embeddings=return_embeddings)
                break
            except spmd.MetaKindChanged:
                self._meta_kind.pop(index_id, None)
                if attempt:
                    raise
            except spmd.RangeMetricsDiffer as e:
                raise RuntimeError(self._range_metrics_differ(index_id, e.metrics))
            except spmd.PlaneError as e:
                raise rpc.ServerException(str(e))
        meta = P.tolist() if int_meta else self._exchange_ids_to_meta(index_id, P)
        return (lims, D, meta, embs) if return_embeddings else (lims, D, meta)

    def _search_with_filter_plane(self, query, top_k, index_id, filter_pos, filter_value):
        from . import spmd

        try:
            D, I, cnt, _e, _m = self.plane.search(index_id, query, 3 * top_k, maximize=self.cfg.metric == "dot",
                                                  filter_pos=filter_pos, filter_value=filter_value, k_out=top_k)
        except spmd.PlaneError as e:
            raise rpc.ServerException(str(e))
        meta = self._exchange_ids_to_meta(index_id, I)
        cnt = cnt.tolist()
        out_scores = [np.ascontiguousarray(D[q, :c], dtype=np.float32).reshape(-1, 1) for q, c in enumerate(cnt)]
        out_meta = [meta[q][:c] for q, c in enumerate(cnt)]
        return out_scores, out_meta

    @staticmethod
    def _aggregate_results(results: List[Tuple], topk: int, q_size: int, maximize_metric: bool,
                           return_embeddings: bool):
        """Merge per-shard `(D[nq,k], meta[nq][k], embs)` tuples, in shard order.
        Winners are identified by their position in the concatenation of all shards' results
        (shard-major), which is also the tie-break: among equal scores the earlier shard wins."""
        D_blocks, flat_meta, flat_embs = [], [], []
        for D, meta_rows, embs in results:
            D_blocks.append(np.ascontiguousarray(D, dtype=np.float32))
            flat_meta.extend(itertools.chain.from_iterable(meta_rows))
            if return_embeddings:
                flat_embs.extend(itertools.chain.from_iterable(embs))
        S = len(D_blocks)
        Dall = np.stack(D_blocks)  # [S, nq, k]
        pos = np.arange(S * q_size * topk, dtype=np.int64).reshape(S, q_size, topk)
        outD, outPos = ResultHeap.merge_backend(Dall, pos, maximize_metric)
        # an unfilled slot (fewer than k hits in total) has position -1 -> metadata None
        # (the reference indexes meta[-1] there, quirk B11 of SURVEY.md)
        picked = [[flat_meta[p] if p >= 0 else None for p in row] for row in outPos.tolist()]
        if not return_embeddings:
            return outD, picked
        picked_embs = [[flat_embs[p] if p >= 0 else None for p in row] for row in outPos.tolist()]
        return outD, picked, picked_embs
