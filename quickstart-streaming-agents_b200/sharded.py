"""Row-sharded search across the GPUs of one box.

The path shards naturally (SURVEY.md section 8e): shard g holds the contiguous rows [offset_g, offset_g + n_g) of the
corpus, every GPU sees the whole query block and runs the same single-GPU scan, and there is exactly ONE exchange step --
an all-gather of each shard's packed per-query (score float64, global row int64) lists, k entries per query
(nq*k*16 bytes per rank: 655 KB at nq = 4096, k = 10) -- followed by a k-way merge on every rank.  No all-reduce, no
all-to-all.

Two deployments, both behind the C ABI (include/sa_api.h, "multi-GPU"):

* ``ShardedIndex`` -- one process per GPU (``torchrun``).  ``transport="nccl"`` (default on CUDA): the communicator lives
  inside libsa_b200.so (``sa_comm_create_rank``; torch.distributed only carries the 128-byte NCCL id once) and a search is
  ONE call, ``sa_sharded_search`` / ``sa_sharded_search_host_submit|wait``: scan, merge, all-gather and shard merge are
  enqueued back to back on one stream with no Python in between, and the host-buffer form keeps two batches in flight.
  ``transport="torch"``: the same steps with ``torch.distributed.all_gather_into_tensor`` as the collective -- what the
  CPU tests drive over gloo with an oracle-backed double (``index`` is duck-typed: ``search_hits`` / ``merge_hits``).
* ``MultiGpuIndex`` -- one process driving all GPUs (``sa_comm_create`` = ncclCommInitAll, ``sa_gather_merge``): what
  ``sa_serve --gpus N`` uses.
"""
from __future__ import annotations

import ctypes as C

import numpy as np
import torch
import torch.distributed as dist

from . import capi
from .engine import host_buffers, stage_filters


def shard_bounds(n_total: int, world: int, rank: int) -> tuple[int, int]:
    """Contiguous, balanced row ranges: rank g owns [g*N//G, (g+1)*N//G)."""
    return rank * n_total // world, (rank + 1) * n_total // world


class ShardedIndex:
    """One rank's shard (a ``VectorIndex`` made with its own ``max_k``, at most 64) in a torch.distributed job: every rank
    searches its rows and the per-shard top-k lists are gathered and merged to the global top-k, for any k <= max_k."""

    def __init__(self, index, row_offset: int, group=None, transport: str | None = None):
        self.index = index
        self.row_offset = int(row_offset)
        self.group = group
        self.world = dist.get_world_size(group) if dist.is_initialized() else 1
        self.rank = dist.get_rank(group) if dist.is_initialized() else 0
        if transport is None:
            transport = "nccl" if (hasattr(index, "_h") and self.world > 1) else "torch"
        self.transport = transport
        self._buf = None
        self._comm = None
        self._inflight = {}
        if transport == "nccl" and self.world > 1:
            self._comm = self._create_comm()

    # ------------------------------------------------------------------ communicator inside the C ABI
    def _create_comm(self):
        lib = self.index.lib
        path = capi.bundled_nccl_path()
        if path:
            capi.check(lib.sa_comm_set_library(path.encode()), "sa_comm_set_library")
        ident = (C.c_char * capi.SA_COMM_ID_BYTES)()
        if self.rank == 0:
            capi.check(lib.sa_comm_unique_id(ident), "sa_comm_unique_id")
        box = [bytes(ident)]
        dist.broadcast_object_list(box, src=dist.get_global_rank(self.group, 0) if self.group is not None else 0,
                                   group=self.group)
        ident = (C.c_char * capi.SA_COMM_ID_BYTES).from_buffer_copy(box[0])
        h = C.c_void_p()
        capi.check(lib.sa_comm_create_rank(C.byref(h), self.world, self.rank, ident, self.index.device),
                   "sa_comm_create_rank")
        return h

    def close(self) -> None:
        if self._comm is not None:
            self.index.lib.sa_comm_destroy(self._comm)
            self._comm = None

    @property
    def dim(self) -> int:
        return self.index.dim

    @property
    def similarity(self) -> str:
        return getattr(self.index, "similarity", "cosine")

    @property
    def dtype(self) -> str:
        """The element type of every rank's index ("bfloat16" for an index that does not say)."""
        return getattr(self.index, "dtype", "bfloat16")

    # ------------------------------------------------------------------ device-resident queries
    def search(self, q: torch.Tensor, k: int, filters=None):
        """q: [nq, dim] of the index's dtype (bf16 or int8) on this rank's device (identical on every rank).  Returns (score f32 [nq,k],
        global row i64 [nq,k]) -- the same on every rank.  ``filters`` (uint64 [nq, 4] or [4], the same on every rank)
        restricts each query to the rows whose tag passes its filter; each rank's index holds its own rows' tags."""
        nq = q.shape[0]
        if self._comm is not None:
            ix = self.index
            q = q.contiguous()
            score = torch.empty((nq, k), dtype=torch.float32, device=q.device)
            rows = torch.empty((nq, k), dtype=torch.int64, device=q.device)
            capi.search(ix.lib, "sa_sharded_search", self._comm, ix._h, q.data_ptr(), nq, k, self.row_offset,
                        score.data_ptr(), rows.data_ptr(), torch.cuda.current_stream(ix.device).cuda_stream,
                        filters=stage_filters(filters, nq, q.device))
            return score, rows
        # an index without filter tags (``search_hits(q, k, row_offset)``) serves the unfiltered searches
        kw = {} if filters is None else {"filters": filters}
        hits = self.index.search_hits(q, k, self.row_offset, **kw)            # uint8 [nq, k, 16]
        if self.world == 1:
            return self.index.merge_hits(hits.view(1, nq, k, 16))
        key = (nq, k, str(hits.device))
        if self._buf is None or self._buf[0] != key:
            self._buf = (key, torch.empty((self.world * nq, k, 16), dtype=torch.uint8, device=hits.device))
        gathered = self._buf[1]
        dist.all_gather_into_tensor(gathered, hits.contiguous(), group=self.group)   # the one collective
        return self.index.merge_hits(gathered.view(self.world, nq, k, 16))

    # ------------------------------------------------------------------ host buffers
    def search_host_submit(self, q_f32: np.ndarray, k: int, slot: int = 0, filters=None) -> None:
        """Enqueue H2D + shard scan + all-gather + merge + D2H for ``slot`` (0 or 1) and return at once."""
        q = np.ascontiguousarray(q_f32, dtype=np.float32)
        if self._comm is None:
            self._inflight[slot] = self._search_host_blocking(q, k, filters)
            return
        ix = self.index
        self._inflight[slot] = (q, q.shape[0], k)   # keeps a pinned source alive until the wait
        capi.search(ix.lib, "sa_sharded_search_host_submit", self._comm, ix._h, slot, q.ctypes.data, q.shape[0], k,
                    self.row_offset, filters=stage_filters(filters, q.shape[0]))

    def search_host_wait(self, slot: int = 0, out=None):
        got = self._inflight.pop(slot)
        if self._comm is None:
            return got
        ix = self.index
        _, nq, k = got
        score, rows = host_buffers(out, nq, k, np.int64)
        capi.check(ix.lib.sa_sharded_search_host_wait(self._comm, ix._h, slot, score.ctypes.data, rows.ctypes.data),
                   "sa_sharded_search_host_wait")
        return score, rows

    def _search_host_blocking(self, q: np.ndarray, k: int, filters=None):
        dev = self.index.rows.device if hasattr(self.index, "rows") else torch.device("cpu")
        if self.dtype == "int8":
            from .engine import int8_round
            qd = torch.from_numpy(int8_round(q)).to(dev)
        else:
            qd = torch.from_numpy(q).to(dev).to(torch.bfloat16)
        s, gi = self.search(qd, k, filters=filters)
        return s.cpu().numpy(), gi.cpu().numpy()

    def search_host(self, q_f32, k: int, out=None, filters=None):
        """Host buffers in, host buffers out (H2D, shard search, all-gather, merge, D2H); blocking."""
        self.search_host_submit(q_f32, k, 0, filters=filters)
        return self.search_host_wait(0, out=out)


class MultiGpuIndex:
    """All GPUs of a box driven by ONE process: shard g of the corpus on device g, one NCCL communicator created inside
    the C ABI (``sa_comm_create``), host queries in and merged host results out through ``sa_gather_merge``.  This is the
    serving form (``sa_serve --gpus N``): no torchrun, no torch.distributed.

    It offers the interface ``operator.VectorTable`` expects of an index (``append`` -> first row, ``delete_rows``,
    ``reset``, ``__len__``, ``search_host[_submit/_wait]``) with DENSE row ids in append order; inside, append batches go
    round-robin to the shards (SURVEY.md section 8e: "append-only streams go round-robin by epoch") and the library's
    global rows (shard * capacity + local row) are translated back through a per-shard table.  ``max_k`` (at most 64,
    ``capi.SA_MAX_K``) is the largest k of a search on every shard; ``similarity`` and ``dtype`` ("bfloat16" or "int8",
    see ``VectorIndex``) are those of every shard."""

    def __init__(self, dim: int, capacity_per_gpu: int, max_batch: int, max_k: int, n_gpus: int | None = None,
                 similarity: str = "cosine", dtype: str = "bfloat16"):
        from .engine import VectorIndex
        n = torch.cuda.device_count() if n_gpus is None else int(n_gpus)
        if n < 1 or n > torch.cuda.device_count():
            raise ValueError(f"n_gpus {n} outside [1, {torch.cuda.device_count()}]")
        self.n = n
        self.dim, self.capacity_per_gpu = dim, int(capacity_per_gpu)
        self.similarity = similarity
        self.dtype = dtype
        self.shards = [VectorIndex(dim=dim, capacity=capacity_per_gpu, max_batch=max_batch, max_k=max_k, device=g,
                                   similarity=similarity, dtype=dtype) for g in range(n)]
        self.lib = self.shards[0].lib
        path = capi.bundled_nccl_path()
        if path:
            capi.check(self.lib.sa_comm_set_library(path.encode()), "sa_comm_set_library")
        h = C.c_void_p()
        devs = (C.c_int * n)(*range(n))
        capi.check(self.lib.sa_comm_create(C.byref(h), n, devs), "sa_comm_create")
        self._comm = h
        self._engines = (C.c_void_p * n)(*[s._h for s in self.shards])
        self._offsets = (C.c_int64 * n)(*[g * self.capacity_per_gpu for g in range(n)])
        self._inflight = {}
        self._next = 0                                    # round-robin appends keep the shards balanced
        self._dense_of = [np.zeros(0, np.int64) for _ in range(n)]   # per shard: local row -> dense row
        self._where: list[tuple[int, int]] = []           # dense row -> (shard, local row)

    def close(self) -> None:
        if self._comm is not None:
            self.lib.sa_comm_destroy(self._comm)
            self._comm = None
        for s in self.shards:
            s.close()

    def __len__(self) -> int:
        return len(self._where)

    def reset(self) -> None:
        for s in self.shards:
            s.reset()
        self._dense_of = [np.zeros(0, np.int64) for _ in range(self.n)]
        self._where = []
        self._next = 0

    def append(self, rows_f32: np.ndarray, tags=None) -> int:
        """Append a batch of fp32 embeddings (int8 ones too, for an int8 index) to the next shard (round-robin).  Returns
        the first (dense) row id.  ``tags`` (uint64 [n]) are the rows' filter tags (0 without)."""
        rows_f32 = np.asarray(rows_f32)
        rows_f32 = np.ascontiguousarray(rows_f32, dtype=np.int8 if rows_f32.dtype == np.int8 else np.float32)
        first = len(self._where)
        if len(rows_f32) == 0:
            return first
        g = self._next
        self._next = (self._next + 1) % self.n
        lo = self.shards[g].append(rows_f32, tags=tags)
        m = len(rows_f32)
        self._dense_of[g] = np.concatenate([self._dense_of[g], np.arange(first, first + m, dtype=np.int64)])
        self._where.extend((g, lo + j) for j in range(m))
        return first

    def delete_rows(self, rows) -> None:
        by_shard: dict[int, list[int]] = {}
        for r in rows:
            g, l = self._where[int(r)]
            by_shard.setdefault(g, []).append(l)
        for g, ls in by_shard.items():
            self.shards[g].delete_rows(ls)

    def set_tags(self, rows, tags) -> None:
        """Rewrite the filter tags of committed (dense) rows; each shard gets its own rows' tags."""
        tags = np.ascontiguousarray(tags, dtype=np.uint64)
        by_shard: dict[int, tuple[list[int], list[int]]] = {}
        for r, t in zip(rows, tags):
            g, l = self._where[int(r)]
            ls, ts = by_shard.setdefault(g, ([], []))
            ls.append(l)
            ts.append(t)
        for g, (ls, ts) in by_shard.items():
            self.shards[g].set_tags(ls, np.array(ts, dtype=np.uint64))

    def _to_dense(self, global_rows: np.ndarray) -> np.ndarray:
        out = np.full(global_rows.shape, -1, dtype=np.int64)
        ok = global_rows >= 0
        g = global_rows[ok] // self.capacity_per_gpu
        l = global_rows[ok] % self.capacity_per_gpu
        dense = np.empty(len(g), dtype=np.int64)
        for s in range(self.n):
            m = g == s
            if m.any():
                dense[m] = self._dense_of[s][l[m]]
        out[ok] = dense
        return out

    def search_host_submit(self, q_f32: np.ndarray, k: int, slot: int = 0, filters=None) -> None:
        """``filters`` (uint64 [nq, 4] or [4]) applies to every shard, each filtering its rows by its own tags."""
        q = np.ascontiguousarray(q_f32, dtype=np.float32)
        self._inflight[slot] = (q, q.shape[0], k)
        capi.search(self.lib, "sa_gather_merge_submit", self._comm, self._engines, slot, q.ctypes.data, q.shape[0], k,
                    self._offsets, filters=stage_filters(filters, q.shape[0]))

    def search_host_wait(self, slot: int = 0, out=None):
        """(score f32 [nq, k], dense row i64 [nq, k]); ties between shards resolve by the library's global row order
        (shard, then local row), not by dense id."""
        _, nq, k = self._inflight.pop(slot)
        score, dense = host_buffers(out, nq, k, np.int64)
        rows = np.empty((nq, k), np.int64)
        capi.check(self.lib.sa_gather_merge_wait(self._comm, self._engines, slot, score.ctypes.data, rows.ctypes.data),
                   "sa_gather_merge_wait")
        dense[:] = self._to_dense(rows)
        return score, dense

    def search_host(self, q_f32: np.ndarray, k: int, out=None, filters=None):
        self.search_host_submit(q_f32, k, 0, filters=filters)
        return self.search_host_wait(0, out=out)
