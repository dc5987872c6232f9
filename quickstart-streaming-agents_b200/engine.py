"""VectorIndex -- the host-side handle of one corpus shard on one H100.

Plays the role of the reference's external vector table ``documents_vectordb_lab2`` (connector 'mongodb',
index 'vector_index', cosine, 1536-d: terraform/lab2-vector-search/main.tf:215,
assets/pre-setup/MongoDB-Setup.md:72-83).  torch tensors are used only as device-memory holders; every
operation is a call into libsa_b200.so through ``capi`` (include/sa_api.h).  No CPU fallback.
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass

import numpy as np
import torch

from . import capi


@dataclass
class SearchTiming:
    scan_ms: float      # sum of the scan-kernel launches of the last search (CUDA events)
    total_ms: float     # first scan start .. last merge end
    bytes: float        # algorithmic bytes of that search
    flops: float        # algorithmic flops of that search
    launches: int       # scan launches
    kernels: int        # all kernels launched


def _ptr(t: torch.Tensor | None) -> int:
    return 0 if t is None else t.data_ptr()


HIT_DTYPE = np.dtype([("score", "<f8"), ("row", "<i8")])   # sa_hit of include/sa_api.h


def filter_array(filters, nq: int) -> np.ndarray:
    """Per-query filters (sa_filter of include/sa_api.h: all_of, none_of, any_of[0], any_of[1]) as a contiguous uint64
    array [nq, 4]; one filter of shape [4] applies to every query."""
    f = np.asarray(filters)
    if f.dtype.kind not in "iu":
        raise TypeError("filters must be an integer array of uint64 words")
    f = f.astype(np.uint64) if f.dtype != np.uint64 else f
    if f.shape == (4,):
        f = np.broadcast_to(f, (nq, 4))
    if f.shape != (nq, 4):
        raise ValueError(f"filters must have shape [4] or [nq={nq}, 4], not {list(f.shape)}")
    return np.ascontiguousarray(f)


def stage_filters(filters, nq: int, device: torch.device | None = None):
    """A search's ``filters`` where the library reads them: for a host call (``device`` None) the numpy array of
    ``filter_array``; for a device call an int64 [nq, 4] tensor on ``device``.  Filters already staged there -- an
    int64 [nq, 4] contiguous CUDA tensor on ``device`` -- are used as is, so a caller can stage them once for many
    searches.  None (an unfiltered search) stays None."""
    if not (isinstance(filters, torch.Tensor) and filters.is_cuda):
        f = None if filters is None else filter_array(filters, nq)
        return f if f is None or device is None else torch.from_numpy(f.view(np.int64).copy()).to(device)
    if filters.device != (None if device is None else torch.device(device)):
        raise ValueError(f"filters on {filters.device} cannot serve a search of queries on {device or 'the host'}")
    if filters.dtype != torch.int64:
        raise TypeError(f"device filters must be an int64 tensor of uint64 words, not {filters.dtype}")
    if tuple(filters.shape) != (nq, 4) or not filters.is_contiguous():
        raise ValueError(f"device filters must be a contiguous [nq={nq}, 4] tensor, not {list(filters.shape)}")
    return filters


def host_buffers(out, nq: int, k: int, idx_dtype=np.int32):
    """The (score f32 [nq, k], idx [nq, k]) host buffers of a search: new arrays, or the caller's ``out`` once checked."""
    if out is None:
        return np.empty((nq, k), np.float32), np.empty((nq, k), idx_dtype)
    score, idx = out
    assert score.shape == (nq, k) and score.dtype == np.float32 and score.flags.c_contiguous
    assert idx.shape == (nq, k) and idx.dtype == idx_dtype and idx.flags.c_contiguous
    return score, idx


def int8_round(x) -> np.ndarray:
    """fp32 -> int8 by the rule every int8 index applies to float input (sa_debug_int8_round): round to nearest even,
    saturate to [-128, 127], NaN -> 0."""
    x = np.ascontiguousarray(x, dtype=np.float32)
    out = np.empty(x.shape, np.int8)
    lib = capi.load()
    capi.check(lib.sa_debug_int8_round(x.ctypes.data, x.size, out.ctypes.data), "sa_debug_int8_round")
    return out


# an index's dtype -> the torch dtype of its rows and of its device queries
TORCH_DTYPES = {"bfloat16": torch.bfloat16, "int8": torch.int8}


def pinned_array(shape, dtype=np.float32) -> np.ndarray:
    """A page-locked numpy array (sa_host_alloc), freed (sa_host_free) when its last view is garbage-collected."""
    import weakref
    lib = capi.load()
    nbytes = int(np.prod(shape)) * np.dtype(dtype).itemsize
    p = C.c_void_p()
    capi.check(lib.sa_host_alloc(C.byref(p), max(nbytes, 1)), "sa_host_alloc")
    buf = (C.c_char * nbytes).from_address(p.value)
    weakref.finalize(buf, lib.sa_host_free, C.c_void_p(p.value))
    return np.frombuffer(buf, dtype=dtype).reshape(shape)


class VectorIndex:
    """A row shard of the corpus resident in HBM: bf16 (or int8) rows [capacity, dim] + one fp32 row term per row
    [capacity].

    ``dtype`` is the element type, fixed at creation: "bfloat16" (default) or "int8" (include/sa_api.h, SA_ELEM_*).  An
    int8 index stores ``rows`` as int8, searches int8 (or fp32) queries and evaluates the similarity on the integers
    themselves, exactly; fp32 input is rounded to nearest even and saturated to [-128, 127] (``int8_round``).  Its
    ``dim`` must be a multiple of 128.

    ``similarity`` is the Atlas index setting, fixed at creation: "cosine" (default), "dotProduct" or "euclidean"
    (include/sa_api.h, SA_SIM_*).  Scores are cosines, dot products or Euclidean distances accordingly; results are
    ordered best first (ascending distance for "euclidean").  ``inv_norm`` holds the row terms: 1/|c| for cosine, 1 for
    dotProduct, |c|^2/2 for euclidean.

    ``max_k`` is the largest k a search may ask for, at most 64 (``capi.SA_MAX_K``); a search with k > 28 runs the deep
    scan variant and is exact like any other.

    ``tags`` holds one 64-bit filter tag per row (uint64 bits in an int64 tensor [capacity]); the searches' ``filters``
    argument restricts each query to the rows whose tag passes its filter (``filter_array``, qsa_b200.filters)."""

    def __init__(self, dim: int = 1536, capacity: int = 1 << 20, max_batch: int = 1024, max_k: int = 10,
                 device: int | None = None, similarity: str = "cosine", dtype: str = "bfloat16"):
        sim = capi.similarity_code(similarity)
        elem = capi.elem_code(dtype)
        if not torch.cuda.is_available():
            raise RuntimeError("VectorIndex needs a CUDA device (H100, sm_90a); there is no CPU fallback")
        self.similarity = similarity
        self.dtype = dtype
        self.lib = capi.load()
        self.device = torch.cuda.current_device() if device is None else int(device)
        self.dim, self.capacity, self.max_batch, self.max_k = int(dim), int(capacity), int(max_batch), int(max_k)
        dev = torch.device("cuda", self.device)
        # device-memory holders (the engine never copies or frees these)
        self.rows = torch.empty((self.capacity, self.dim), dtype=TORCH_DTYPES[dtype], device=dev)
        self.inv_norm = torch.zeros((self.capacity,), dtype=torch.float32, device=dev)
        self.tags = torch.zeros((self.capacity,), dtype=torch.int64, device=dev)
        h = C.c_void_p()
        capi.check(self.lib.sa_engine_create_elem(C.byref(h), self.device, self.dim, self.capacity, self.max_batch,
                                                  self.max_k, sim, elem), "sa_engine_create_elem")
        self._h = h
        self._inflight = {}
        capi.check(self.lib.sa_corpus_bind(self._h, self.rows.data_ptr(), self.inv_norm.data_ptr(), 0),
                   "sa_corpus_bind")
        capi.check(self.lib.sa_corpus_bind_tags(self._h, self.tags.data_ptr()), "sa_corpus_bind_tags")

    # ------------------------------------------------------------------ lifecycle
    def close(self) -> None:
        """Destroy the engine.  Page-locked arrays handed out by ``pinned_array`` are NOT freed here: each is released
        when its last numpy view is garbage-collected, so a caller still holding one never touches freed memory."""
        if getattr(self, "_h", None):
            self.lib.sa_engine_destroy(self._h)
            self._h = None

    def __del__(self):  # pragma: no cover
        try:
            self.close()
        except Exception:
            pass

    def __len__(self) -> int:
        return int(self.lib.sa_corpus_rows(self._h))

    def _stream(self) -> int:
        return torch.cuda.current_stream(self.device).cuda_stream

    def set_option(self, name: str, value: int) -> None:
        capi.check(self.lib.sa_set_option(self._h, name.encode(), int(value)), "sa_set_option")

    def info(self, name: str) -> int:
        v = C.c_int64()
        capi.check(self.lib.sa_get_info(self._h, name.encode(), C.byref(v)), "sa_get_info")
        return int(v.value)

    # ------------------------------------------------------------------ ingest
    def reset(self) -> None:
        """Forget every row (the job of scripts/common/clear_mongodb.py:98-158 in the reference)."""
        capi.check(self.lib.sa_corpus_reset(self._h), "sa_corpus_reset")

    def _write_tags(self, first: int, n: int, tags) -> None:
        """Tags of rows [first, first + n): the given uint64 words, or zeros.  Written before the rows are committed."""
        if first + n > self.capacity:
            raise capi.SaError(capi.SA_ERR_CAPACITY, "tags", "append past capacity")
        if tags is None:
            self.tags[first:first + n].zero_()
            return
        t = np.ascontiguousarray(tags, dtype=np.uint64)
        if t.shape != (n,):
            raise ValueError(f"tags must have shape [{n}], not {list(t.shape)}")
        self.tags[first:first + n].copy_(torch.from_numpy(t.view(np.int64)))

    def set_tags(self, rows, tags) -> None:
        """Rewrite the tags of committed rows (between searches)."""
        ix = torch.as_tensor(np.asarray(rows, dtype=np.int64), device=self.tags.device)
        t = np.ascontiguousarray(tags, dtype=np.uint64)
        if t.shape != (len(ix),):
            raise ValueError(f"tags must have shape [{len(ix)}], not {list(t.shape)}")
        if len(ix) and (int(ix.min()) < 0 or int(ix.max()) >= len(self)):
            raise IndexError("set_tags: row outside the committed rows")
        self.tags[ix] = torch.from_numpy(t.view(np.int64)).to(self.tags.device)

    def append(self, rows_f32, tags=None) -> int:
        """Append fp32 embeddings (host numpy or device tensor) -> bf16 (or int8) rows + row terms.  Returns first row
        id.  An int8 index also takes int8 rows (numpy or CUDA tensor), stored exactly as given.
        ``tags`` (uint64 [n]) are the new rows' filter tags; without them the rows get tag 0."""
        first = len(self)
        is_t = isinstance(rows_f32, torch.Tensor)
        if self.dtype == "int8" and (rows_f32.dtype == torch.int8 if is_t else np.asarray(rows_f32).dtype == np.int8):
            return self._append_in_place(rows_f32, tags)
        if isinstance(rows_f32, torch.Tensor) and rows_f32.is_cuda:
            x = rows_f32.to(torch.float32).contiguous()
            assert x.dim() == 2 and x.shape[1] == self.dim
            self._write_tags(first, x.shape[0], tags)
            capi.check(self.lib.sa_corpus_append_f32(self._h, x.data_ptr(), x.shape[0], self._stream()),
                       "sa_corpus_append_f32")
            torch.cuda.current_stream(self.device).synchronize()  # x may be freed by the caller
        else:
            x = np.ascontiguousarray(rows_f32, dtype=np.float32)
            assert x.ndim == 2 and x.shape[1] == self.dim
            self._write_tags(first, x.shape[0], tags)
            torch.cuda.current_stream(self.device).synchronize()  # the *_host calls run on the engine's stream
            capi.check(self.lib.sa_corpus_append_host_f32(self._h, x.ctypes.data, x.shape[0]),
                       "sa_corpus_append_host_f32")
        return first

    def append_bf16_bits(self, bits: np.ndarray, tags=None) -> int:
        """Append rows given as bf16 bit patterns (uint16 [n, dim]) -- used with the synthetic corpora so the
        device holds exactly the bits the oracle sees.  ``tags`` as in ``append``.  Not for an int8 index."""
        if self.dtype != "bfloat16":
            raise TypeError(f"append_bf16_bits needs a bfloat16 index; this one is {self.dtype}")
        bits = np.ascontiguousarray(bits, dtype=np.uint16)
        return self._append_in_place(torch.from_numpy(bits.view(np.int16)).view(torch.bfloat16), tags)

    def _append_in_place(self, src, tags=None) -> int:
        """Rows already of the index's element type (numpy or tensor [n, dim]) written into ``rows`` and committed."""
        src = torch.from_numpy(np.ascontiguousarray(src)) if isinstance(src, np.ndarray) else src
        assert src.dim() == 2 and src.shape[1] == self.dim and src.dtype == self.rows.dtype
        first = len(self)
        n = src.shape[0]
        if first + n > self.capacity:
            raise capi.SaError(capi.SA_ERR_CAPACITY, "append", "append past capacity")
        self._write_tags(first, n, tags)
        self.rows[first:first + n].copy_(src)
        self.commit(first, n)
        return first

    # ------------------------------------------------------------------ checkpoint / resume
    def snapshot(self, path: str) -> int:
        """Write the committed rows (bf16 bits, or int8), their row terms, their filter tags, the similarity and the
        dtype to ``path`` (.npz).  Returns the row count.
        (The reference leaves corpus durability to Atlas; here a snapshot + the consumer-group offsets are the
        checkpoint, and replaying `documents_embed` from offset 0 is the fallback.)"""
        n = len(self)
        torch.cuda.current_stream(self.device).synchronize()
        if self.dtype == "int8":
            bits = self.rows[:n].cpu().numpy()
        else:
            bits = self.rows[:n].view(torch.int16).cpu().numpy().view(np.uint16)
        import os
        path = path if path.endswith(".npz") else path + ".npz"
        tmp = path + ".tmp"
        with open(tmp, "wb") as f:                       # written under a temporary name, then renamed: never half a file
            np.savez(f, rows=bits, inv_norm=self.inv_norm[:n].cpu().numpy(), dim=np.int64(self.dim),
                     similarity=np.str_(self.similarity), tags=self.tags[:n].cpu().numpy().view(np.uint64),
                     dtype=np.str_(self.dtype))
            f.flush()
            os.fsync(f.fileno())
        os.replace(tmp, path)
        return n

    def restore(self, path: str) -> int:
        """Load a snapshot written by ``snapshot`` into this (empty or not) index, replacing its contents.  A snapshot
        without a recorded similarity is a cosine one; a snapshot of another similarity is refused (its row terms and
        its rankings mean something else).  A snapshot without tags restores tag 0 on every row.  Likewise a snapshot
        that does not name a dtype is a bfloat16 one, and a snapshot of the other dtype is refused."""
        z = np.load(path if path.endswith(".npz") else path + ".npz")
        if int(z["dim"]) != self.dim:
            raise ValueError(f"snapshot has dim {int(z['dim'])}, index has {self.dim}")
        snap_sim = str(z["similarity"]) if "similarity" in z.files else "cosine"
        if snap_sim != self.similarity:
            raise ValueError(f"snapshot has similarity {snap_sim!r}, index has {self.similarity!r}")
        snap_dtype = str(z["dtype"]) if "dtype" in z.files else "bfloat16"
        if snap_dtype != self.dtype:
            raise ValueError(f"snapshot has dtype {snap_dtype!r}, index has {self.dtype!r}")
        bits, inv = z["rows"], z["inv_norm"]
        n = bits.shape[0]
        if n > self.capacity:
            raise capi.SaError(capi.SA_ERR_CAPACITY, "restore", "snapshot larger than capacity")
        if self.dtype == "int8":
            self.rows[:n].copy_(torch.from_numpy(np.ascontiguousarray(bits, dtype=np.int8)))
        else:
            self.rows[:n].copy_(torch.from_numpy(bits.view(np.int16)).view(torch.bfloat16))
        self.inv_norm[:n].copy_(torch.from_numpy(inv))
        if "tags" in z.files:
            self.tags[:n].copy_(torch.from_numpy(np.ascontiguousarray(z["tags"], dtype=np.uint64).view(np.int64)))
        else:
            self.tags[:n].zero_()
        torch.cuda.current_stream(self.device).synchronize()
        capi.check(self.lib.sa_corpus_bind(self._h, self.rows.data_ptr(), self.inv_norm.data_ptr(), n),
                   "sa_corpus_bind")
        return n

    def delete_rows(self, rows) -> None:
        """Tombstone rows: zero the stored vector and write the tombstone row term (0, or -1 for euclidean, where a
        zero vector is a live row) -- tombstoned rows are never returned."""
        if len(rows) == 0:
            return
        ix = torch.as_tensor(list(rows), dtype=torch.long, device=self.rows.device)
        self.rows.index_fill_(0, ix, 0)
        self.inv_norm.index_fill_(0, ix, -1.0 if self.similarity == "euclidean" else 0.0)

    def commit(self, first: int, n: int) -> None:
        """Rows [first, first+n) were written into ``self.rows`` in place: compute norms and publish them."""
        capi.check(self.lib.sa_corpus_commit(self._h, int(first), int(n), self._stream()), "sa_corpus_commit")

    # ------------------------------------------------------------------ search
    def search(self, q: torch.Tensor, k: int, want_score64: bool = False, filters=None):
        """Device path.  q: [nq, dim] CUDA tensor of the index's dtype (bf16 or int8) or fp32.  Returns (score f32 [nq,k], idx i32 [nq,k]
        [, score64 f64 [nq,k]]) as CUDA tensors, asynchronous on the current stream.  ``filters`` (uint64 [nq, 4] or
        [4], see ``filter_array``, or an int64 [nq, 4] tensor on q's device, see ``stage_filters``) restricts each query
        to the rows whose tag passes its filter."""
        assert q.is_cuda and q.dim() == 2 and q.shape[1] == self.dim
        name = {self.rows.dtype: "sa_search", torch.float32: "sa_search_f32"}.get(q.dtype)
        if name is None:
            raise TypeError(f"queries of a {self.dtype} index must be {self.dtype} or fp32, not {q.dtype}")
        q = q.contiguous()
        nq = q.shape[0]
        dev = q.device
        score = torch.empty((nq, k), dtype=torch.float32, device=dev)
        idx = torch.empty((nq, k), dtype=torch.int32, device=dev)
        s64 = torch.empty((nq, k), dtype=torch.float64, device=dev) if want_score64 else None
        capi.search(self.lib, name, self._h, q.data_ptr(), nq, k, score.data_ptr(), idx.data_ptr(), _ptr(s64),
                    self._stream(), filters=stage_filters(filters, nq, dev))
        return (score, idx, s64) if want_score64 else (score, idx)

    def search_host(self, q_f32: np.ndarray, k: int, out=None, filters=None):
        """End-to-end path with HOST buffers (H2D, search, D2H inside the call).  Returns numpy
        (score f32 [nq,k], idx i32 [nq,k]); ``out=(score, idx)`` reuses caller buffers (e.g. ``pinned_array``).
        ``filters`` as in ``search``, as a host array."""
        q = np.ascontiguousarray(q_f32, dtype=np.float32)
        assert q.ndim == 2 and q.shape[1] == self.dim
        nq = q.shape[0]
        score, idx = host_buffers(out, nq, k)
        torch.cuda.current_stream(self.device).synchronize()  # the *_host calls run on the engine's stream
        capi.search(self.lib, "sa_search_host", self._h, q.ctypes.data, nq, k, score.ctypes.data, idx.ctypes.data,
                    filters=stage_filters(filters, nq))
        return score, idx

    def search_host_submit(self, q_f32: np.ndarray, k: int, slot: int = 0, filters=None) -> None:
        """First half of ``search_host``: enqueue H2D + search + D2H for ``slot`` (0 or 1) and return at once, so the
        caller can prepare the next batch while the GPU works.  Collect with ``search_host_wait(slot)``.
        ``filters`` as in ``search_host`` (staged by the call: the array may be reused at once)."""
        q = np.ascontiguousarray(q_f32, dtype=np.float32)
        assert q.ndim == 2 and q.shape[1] == self.dim
        torch.cuda.current_stream(self.device).synchronize()  # the *_host calls run on the engine's own stream
        self._inflight[slot] = (q, q.shape[0], k)  # keeps a pinned source alive until the wait
        capi.search(self.lib, "sa_search_host_submit", self._h, slot, q.ctypes.data, q.shape[0], k,
                    filters=stage_filters(filters, q.shape[0]))

    def search_host_wait(self, slot: int = 0, out=None):
        _, nq, k = self._inflight.pop(slot)
        score, idx = host_buffers(out, nq, k)
        capi.check(self.lib.sa_search_host_wait(self._h, slot, score.ctypes.data, idx.ctypes.data),
                   "sa_search_host_wait")
        return score, idx

    def pinned_array(self, shape, dtype=np.float32) -> np.ndarray:
        """A page-locked numpy array (sa_host_alloc): passing such buffers to ``search_host`` lets the engine DMA
        them directly instead of staging through its own pinned copy.  Freed when its last view is garbage-collected,
        not when the index is closed (see ``close``)."""
        return pinned_array(shape, dtype)

    def search_hits(self, q: torch.Tensor, k: int, row_offset: int = 0, filters=None) -> torch.Tensor:
        """This shard's results in exchange format: uint8 CUDA tensor [nq, k, 16] = sa_hit {score f64, global row i64}
        (``hits.view(torch.float64)[..., 0]`` / ``.view(torch.int64)[..., 1]``).  q: the index's dtype.  ``filters`` as
        in ``search``."""
        assert q.is_cuda and q.dtype == self.rows.dtype and q.dim() == 2 and q.shape[1] == self.dim
        q = q.contiguous()
        hits = torch.empty((q.shape[0], k, 16), dtype=torch.uint8, device=q.device)
        capi.search(self.lib, "sa_search_hits", self._h, q.data_ptr(), q.shape[0], k, int(row_offset), hits.data_ptr(),
                    self._stream(), filters=stage_filters(filters, q.shape[0], q.device))
        return hits

    def merge_hits(self, hits_all: torch.Tensor):
        """hits_all: uint8 [n_shards, nq, k, 16] gathered from all shards.  Returns (score f32 [nq,k], global row i64)."""
        g, nq, k, _ = hits_all.shape
        score = torch.empty((nq, k), dtype=torch.float32, device=hits_all.device)
        idx = torch.empty((nq, k), dtype=torch.int64, device=hits_all.device)
        capi.check(self.lib.sa_merge_hits(self._h, hits_all.contiguous().data_ptr(), g, nq, k, score.data_ptr(),
                                          idx.data_ptr(), self._stream()), "sa_merge_hits")
        return score, idx

    def scan_profile(self) -> dict:
        """Per-CTA role counters of the last scan launch run with option "profile" = 1 (SM cycles): how long the TMA
        producer waited for a free smem slot, the MMA issuer for data / for the epilogue, the epilogue for the MMA, and
        how long the epilogue worked.  Arrays are indexed by CTA."""
        n = self.info("last_grid")
        a = np.zeros((n, 8), dtype=np.int64)
        got = C.c_int()
        capi.check(self.lib.sa_scan_profile(self._h, a.ctypes.data, n, C.byref(got)), "sa_scan_profile")
        a = a[:got.value]
        names = ("prod_wait_empty", "mma_wait_full", "mma_wait_tempty", "epi_wait_tfull", "epi_busy", "epi_slow_chunks",
                 "total", "tiles")
        return {nm: a[:, i] for i, nm in enumerate(names)}

    def merge_shards(self, score64_all: torch.Tensor, gidx_all: torch.Tensor):
        """score64_all / gidx_all: [n_shards, nq, k] (float64 / int64 global rows) gathered from all ranks.
        Returns (score f32 [nq,k], global idx i64 [nq,k])."""
        g, nq, k = score64_all.shape
        score = torch.empty((nq, k), dtype=torch.float32, device=score64_all.device)
        idx = torch.empty((nq, k), dtype=torch.int64, device=score64_all.device)
        capi.check(self.lib.sa_merge_shards(self._h, score64_all.contiguous().data_ptr(),
                                            gidx_all.contiguous().data_ptr(), g, nq, k, score.data_ptr(),
                                            idx.data_ptr(), self._stream()), "sa_merge_shards")
        return score, idx

    def last_timing(self) -> SearchTiming:
        a, b = C.c_float(), C.c_float()
        by, fl = C.c_double(), C.c_double()
        n, kn = C.c_int(), C.c_int()
        capi.check(self.lib.sa_last_timing(self._h, C.byref(a), C.byref(b), C.byref(by), C.byref(fl), C.byref(n),
                                           C.byref(kn)), "sa_last_timing")
        return SearchTiming(a.value, b.value, by.value, fl.value, n.value, kn.value)

    def timing_mean(self, n: int = 16) -> tuple[float, float, int]:
        """(mean scan ms, mean total ms, searches averaged) over the most recent min(n, 16) searches."""
        a, b, m = C.c_float(), C.c_float(), C.c_int()
        capi.check(self.lib.sa_timing_mean(self._h, int(n), C.byref(a), C.byref(b), C.byref(m)), "sa_timing_mean")
        return a.value, b.value, m.value

    def debug_tile_dots(self, q_bf16: torch.Tensor, tile: int, cta_group: int = 1) -> torch.Tensor:
        """Test hook: raw Q.C^T accumulators of one 256-row corpus tile, [padded nq, 256] fp32 (int8: the exact int32
        accumulators rounded to fp32).  q: the index's dtype."""
        assert q_bf16.dtype == self.rows.dtype
        nq = q_bf16.shape[0]
        rows = 128 * cta_group
        padded = (nq + rows - 1) // rows * rows
        out = torch.zeros((padded, 256), dtype=torch.float32, device=q_bf16.device)
        capi.check(self.lib.sa_debug_tile_dots(self._h, q_bf16.contiguous().data_ptr(), nq, tile, cta_group,
                                               out.data_ptr(), self._stream()), "sa_debug_tile_dots")
        return out
