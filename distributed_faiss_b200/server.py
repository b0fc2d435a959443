"""IndexServer: one rank = one shard process = one H100.

API mirror of the reference's `IndexServer` (distributed_faiss/server.py:38-404): same
constructor, same remotely callable method names (dispatch by name, server.py:224-229),
same `{storage_dir}/{index_id}/{rank}/` layout (server.py:382-388), same error convention
(exception -> traceback text -> rpc.ServerException on the client, server.py:229-236).
Rank r is pinned to GPU r % visible_devices; every Index it owns keeps its vectors in that
GPU's HBM (engine.GpuIndex).
"""
import logging
import os
import pathlib
import socket
import sys
import threading
import traceback
from typing import Callable, List, Optional, Tuple

import numpy as np

from .index import Index
from .index_cfg import IndexCfg
from .index_state import IndexState
from .rpc import DEFAULT_PORT, ClientExit, recv_msg, send_msg

logger = logging.getLogger("distributed_faiss_b200")


class IndexServer:
    def __init__(self, rank: int, index_storage_dir, engine_factory: Optional[Callable] = None,
                 device: Optional[int] = None):
        self.indexes = {}
        self.indexes_lock = threading.Lock()
        self.rank = rank
        self.socket = None
        self.index_storage_dir = index_storage_dir
        self._engine_factory = engine_factory
        self._stopping = False
        # GPU ordinal of this rank; settable before the first index is created (one process that
        # hosts several server ranks on one GPU, e.g. the 1-GPU point of the scaling curve)
        self.device = device

    # ------------------------------------------------------------ device pinning
    def _device(self):
        """rank r -> GPU r (mod visible devices); None when an engine factory is injected / no GPU"""
        if self._engine_factory is not None:
            return None
        import torch

        if not torch.cuda.is_available():
            return None
        if self.device is None:
            self.device = self.rank % torch.cuda.device_count()
        return self.device

    def _bind_device(self):
        dev = self._device()
        if dev is not None:
            import torch

            torch.cuda.set_device(dev)

    # ------------------------------------------------------------ service loop
    def start_blocking(self, port=DEFAULT_PORT, v6=False, load_index=False):
        if load_index:
            self.load_index()
        family = socket.AF_INET6 if v6 else socket.AF_INET
        s = socket.socket(family, socket.SOCK_STREAM)
        s.setsockopt(socket.SOL_SOCKET, socket.SO_REUSEADDR, 1)
        s.bind(("", port))
        s.listen(64)
        self.socket = s
        while not self._stopping:
            try:
                conn, _addr = s.accept()
            except OSError:
                if self._stopping:
                    break
                raise
            conn.setsockopt(socket.IPPROTO_TCP, socket.TCP_NODELAY, 1)
            threading.Thread(target=self.exec_loop_blocking, args=(conn,), daemon=True).start()

    def start(self, port=DEFAULT_PORT, v6=False):
        """Non-blocking flavour of the reference (server.py:137): serve from a daemon thread."""
        t = threading.Thread(target=self.start_blocking, args=(port, v6), daemon=True)
        t.start()
        return t

    def exec_loop_blocking(self, conn):
        self._bind_device()
        try:
            while True:
                self.one_function_blocking(conn)
        except (ClientExit, ConnectionError, OSError):
            pass
        except BaseException:
            traceback.print_exc(50, sys.stderr)
        finally:
            try:
                conn.close()
            except OSError:
                pass

    def one_function_blocking(self, conn):
        fname, args = recv_msg(conn)
        st, ret = None, None
        try:
            fn = getattr(self, fname)
        except AttributeError:
            fn = None
            st = "unknown method " + fname
        if fn is not None:
            try:
                ret = fn(*args)
            except Exception as e:  # forwarded to the caller, as the reference does
                st = "".join(traceback.format_tb(sys.exc_info()[2])) + str(e)
        send_msg(conn, (st, ret))

    def stop(self):
        self._stopping = True
        if self.socket:
            try:
                self.socket.shutdown(socket.SHUT_RDWR)
            except OSError:
                pass
            self.socket.close()
            self.socket = None
        for index in list(self.indexes.values()):
            index.save()

    # ------------------------------------------------------------ remotely callable methods
    def get_rank(self) -> int:
        return self.rank

    def create_index(self, index_id: str, cfg: IndexCfg):
        self._bind_device()
        cfg.index_storage_dir = self._get_storage_dir(index_id, cfg)
        pathlib.Path(cfg.index_storage_dir).mkdir(parents=True, exist_ok=True)
        with self.indexes_lock:
            if index_id in self.indexes:
                return False
            self.indexes[index_id] = Index(cfg, engine_factory=self._engine_factory, device=self._device())
            return True

    def add_index_data(self, index_id: str, embeddings: np.ndarray, metadata: Optional[List[object]] = None,
                       train_async_if_triggered: bool = True):
        with self.indexes_lock:
            index = self.indexes[index_id]
        index.add_batch(embeddings, metadata, train_async_if_triggered)

    def sync_train(self, index_id: str):
        self._get_index(index_id).train()

    def async_train(self, index_id: str):
        # the reference runs this synchronously too (it calls Thread.run, server.py:317-318)
        self._get_index(index_id).train()

    def search(self, index_id: str, query_batch: np.ndarray, top_k: int, return_embeddings: bool) -> Tuple:
        return self._get_index(index_id).search(query_batch, top_k=top_k, return_embeddings=return_embeddings)

    def range_search(self, index_id: str, query_batch: np.ndarray, radius: float,
                     return_embeddings: bool = False) -> Tuple:
        """(lims, scores, meta, search metric) of this shard, and with `return_embeddings` the hits'
        vectors float32[lims[-1], d] as a fifth item; IndexClient.range_search merges them"""
        index = self._get_index(index_id)
        lims, scores, meta, *embs = index.range_search(query_batch, radius, return_embeddings)
        return (lims, scores, meta, index.search_metric(), *embs)

    def search_ids(self, index_id: str, query_batch: np.ndarray, top_k: int):
        return self._get_index(index_id).search_ids(query_batch, top_k)

    # ---- support of the NCCL data plane (spmd.SearchPlane); control-plane calls, not timed
    def adopt_index(self, index_id: str, cfg: IndexCfg, engine, meta_table=None) -> None:
        """register a shard built directly on this rank's GPU (in-process callers only)"""
        self._bind_device()
        cfg.index_storage_dir = self._get_storage_dir(index_id, cfg)
        index = Index(cfg, engine_factory=self._engine_factory, device=self._device())
        index.adopt_engine(engine, meta_table)
        with self.indexes_lock:
            self.indexes[index_id] = index

    def get_meta_kind(self, index_id: str) -> str:
        return self._get_index(index_id).get_meta_kind()

    def lookup_meta(self, index_id: str, local_ids) -> List[object]:
        return self._get_index(index_id).lookup_meta(local_ids)

    def get_centroids(self, index_id: str):
        return self._get_index(index_id).get_centroids()

    def set_nprobe(self, index_id: str, nprobe: int):
        return self._get_index(index_id).set_nprobe(nprobe)

    def get_state(self, index_id: str):
        return self._get_index(index_id).get_state()

    def add_buffer_to_index(self, index_id: str):
        return self._get_index(index_id).add_buffer_to_index()

    def get_ntotal(self, index_id: str) -> int:
        with self.indexes_lock:
            index = self.indexes.get(index_id)
        return 0 if index is None else index.get_idx_data_num()[1]

    def get_aggregated_ntotal(self, index_id: str) -> int:
        with self.indexes_lock:
            index = self.indexes[index_id]
        return index.get_idx_data_num()[0]

    def get_ids(self, index_id: str = "default") -> set:
        with self.indexes_lock:
            index = self.indexes[index_id]
        return index.get_ids()

    def index_loaded(self, index_id: str) -> bool:
        with self.indexes_lock:
            index = self.indexes.get(index_id)
        return index is not None and index.get_state() == IndexState.TRAINED

    def drop_index(self, index_id: str):
        with self.indexes_lock:
            index = self.indexes.pop(index_id, None)
        if index is not None:
            index.drop_index()  # releases the engine (HBM) and stops the save watcher

    def save_index(self, index_id: str):
        with self.indexes_lock:
            if index_id not in self.indexes:
                raise RuntimeError(f"Index with id={index_id} is not initialized")
            index = self.indexes[index_id]
        index.save()

    def load_index(self, index_id: str = "default", cfg: IndexCfg = None) -> bool:
        self._bind_device()
        index_dir = self._get_storage_dir(index_id, cfg)
        if cfg:
            cfg.index_storage_dir = index_dir
        with self.indexes_lock:
            if index_id in self.indexes:
                if cfg:
                    self.indexes[index_id].upd_cfg(cfg)
                return True
            index = Index.from_storage_dir(index_dir, cfg, engine_factory=self._engine_factory,
                                           device=self._device())
            if index is None:
                return False
            self.indexes[index_id] = index
            return True

    def get_config_path(self, index_id: str):
        return os.path.join(self.index_storage_dir, index_id, str(self.rank), "cfg.json")

    # ------------------------------------------------------------ helpers
    def _get_index(self, index_id: str) -> Index:
        with self.indexes_lock:
            if index_id not in self.indexes:
                raise RuntimeError("Server has no index with id={}".format(index_id))
            return self.indexes[index_id]

    def _get_storage_dir(self, index_id: str, cfg: IndexCfg):
        base = cfg.index_storage_dir if cfg else None
        if not base:
            return os.path.join(self.index_storage_dir, index_id, str(self.rank))
        return os.path.join(base, str(self.rank))
