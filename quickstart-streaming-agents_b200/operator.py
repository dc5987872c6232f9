"""VECTOR_SEARCH_AGG drop-in.

Reference statement (terraform/lab2-vector-search/main.tf:292)::

    SELECT qe.query, vs.search_results[1].document_id AS document_id_1, vs.search_results[1].chunk AS chunk_1,
           vs.search_results[1].score AS score_1, ... [2] ..., ... [3] ...
    FROM queries_embed AS qe,
         LATERAL TABLE(VECTOR_SEARCH_AGG(documents_vectordb_lab2, DESCRIPTOR(embedding), qe.embedding, 3)) AS vs

``VectorTable`` is the external table ``documents_vectordb_lab2 (document_id STRING, chunk STRING, embedding
ARRAY<FLOAT>)`` (main.tf:215; Lab4 adds metadata columns, terraform/lab4-pubsec-fraud-agents/main.tf:271-289):
the embedding column lives in HBM inside a ``VectorIndex``, the other columns in a host side table.
``vector_search_agg(table, "embedding", query_vectors, k)`` returns, per query, the 1-indexed
``search_results`` array of rows ``(table columns..., score)`` in descending score order.

The index object only needs ``append(rows_f32) -> first_row``, ``search_host(q_f32, k) -> (score, idx)``,
``reset()``, ``__len__`` and ``delete_rows`` -- production passes ``engine.VectorIndex`` (CUDA, no fallback).  A table
with ``filter_fields`` (Atlas's ``{"type": "filter"}`` fields) also needs ``append(rows, tags=...)``, ``set_tags`` and
``search_host(..., filters=...)``.
"""
from __future__ import annotations

from dataclasses import dataclass, field

import numpy as np

from .filters import FilterSchema, compile_filter


def _avro_nullable_string(v: str | None) -> bytes:
    if v is None:
        return b"\x00"
    raw = v.encode("utf-8")
    out = bytearray(b"\x02")
    n = len(raw) << 1  # zig-zag of a non-negative length
    while n > 0x7F:
        out.append((n & 0x7F) | 0x80)
        n >>= 7
    out.append(n)
    return bytes(out) + raw


class ByteArena:
    """Append-only arena of byte strings with an offsets table (value i = data[off[i]:off[i+1]]), kept in numpy
    arrays so the native encoder (sa_wire_encode_search_results) can read it in place."""

    def __init__(self):
        self.data = np.zeros(1 << 16, dtype=np.uint8)
        self.off = np.zeros(1 << 10, dtype=np.uint64)
        self.n = 0
        self.used = 0

    def append(self, b: bytes) -> None:
        need = self.used + len(b)
        if need > self.data.size:
            grown = np.zeros(max(need, 2 * self.data.size), dtype=np.uint8)
            grown[:self.used] = self.data[:self.used]
            self.data = grown
        if self.n + 2 > self.off.size:
            grown = np.zeros(2 * self.off.size, dtype=np.uint64)
            grown[:self.n + 1] = self.off[:self.n + 1]
            self.off = grown
        self.data[self.used:need] = np.frombuffer(b, dtype=np.uint8)
        self.used = need
        self.n += 1
        self.off[self.n] = need

    def extend(self, items: list[bytes]) -> None:
        """Append many values with one copy (what the ingest path uses: a batch at a time)."""
        if not items:
            return
        blob = b"".join(items)
        need = self.used + len(blob)
        if need > self.data.size:
            grown = np.zeros(max(need, 2 * self.data.size), dtype=np.uint8)
            grown[:self.used] = self.data[:self.used]
            self.data = grown
        m = len(items)
        if self.n + m + 1 > self.off.size:
            grown = np.zeros(max(self.n + m + 1, 2 * self.off.size), dtype=np.uint64)
            grown[:self.n + 1] = self.off[:self.n + 1]
            self.off = grown
        self.data[self.used:need] = np.frombuffer(blob, dtype=np.uint8)
        lens = np.fromiter(map(len, items), dtype=np.uint64, count=m)
        self.off[self.n + 1:self.n + m + 1] = np.uint64(self.used) + np.cumsum(lens)
        self.used = need
        self.n += m

    def clear(self) -> None:
        self.n = 0
        self.used = 0


@dataclass
class SearchHit:
    document_id: str | None
    chunk: str | None
    score: float
    row: int
    metadata: dict = field(default_factory=dict)


class VectorTable:
    """``filter_fields``: the metadata columns declared as Atlas filter fields; their values become the rows' tags, and
    ``vector_search_agg(..., filter=...)`` restricts a search to the rows matching an MQL predicate over them."""

    def __init__(self, index, name: str = "documents_vectordb_lab2", embedding_column: str = "embedding",
                 filter_fields=()):
        self.index = index
        self.name = name
        self.embedding_column = embedding_column
        self.filter_fields = tuple(filter_fields)
        self.filter_schema = FilterSchema(self.filter_fields) if self.filter_fields else None
        self.document_id: list[str | None] = []
        self.chunk: list[str | None] = []
        self.metadata: list[dict] = []
        self._row_of: dict[str, int] = {}
        # the string columns pre-serialised as Avro ["null","string"] values (branch byte + length + utf-8): emitting a
        # search_results record is then a concatenation of ready-made byte strings (pipeline/serve.py fast path)
        self.avro_document_id: list[bytes] = []
        self.avro_chunk: list[bytes] = []
        # ... and the same bytes in arenas, for the native batch encoder (sa_wire_encode_search_results)
        self.arena_document_id = ByteArena()
        self.arena_chunk = ByteArena()
        # offsets of the source topic (documents_embed) up to which this table's content is complete; restored by load()
        self.source_offsets: dict[str, int] | None = None

    def _push_avro(self, document_id, chunk) -> None:
        d, c = _avro_nullable_string(document_id), _avro_nullable_string(chunk)
        self.avro_document_id.append(d)
        self.avro_chunk.append(c)
        self.arena_document_id.append(d)
        self.arena_chunk.append(c)

    def __len__(self) -> int:
        return len(self.document_id)

    @property
    def similarity(self) -> str:
        """The index's similarity ("cosine" for an index that does not say)."""
        return index_similarity(self.index)

    def upsert_many(self, document_ids, chunks, embeddings: np.ndarray, metadata=None) -> None:
        """Insert rows; a document_id seen before replaces its old row (sink-connector upsert semantics): the
        old row is tombstoned (``delete_rows``), and tombstoned rows are never returned by the engine."""
        embeddings = np.ascontiguousarray(embeddings, dtype=np.float32)
        n = len(document_ids)
        assert embeddings.shape[0] == n and len(chunks) == n
        metadata = metadata or [{} for _ in range(n)]
        stale = [self._row_of[d] for d in document_ids if d is not None and d in self._row_of]
        # a document repeated inside this very batch: keep its last occurrence only
        last = {d: i for i, d in enumerate(document_ids) if d is not None}
        keep = [i for i, d in enumerate(document_ids) if d is None or last[d] == i]
        rows = embeddings if len(keep) == n else embeddings[keep]
        if self.filter_schema is not None:
            tags = self.filter_schema.tags([metadata[i] for i in keep])   # before anything is mutated: may refuse
        if stale:
            self.index.delete_rows(stale)
        if self.filter_schema is not None:
            first = self.index.append(rows, tags=tags)
        else:
            first = self.index.append(rows)
        assert first == len(self.document_id), "side table and index out of step"
        ids = [document_ids[i] for i in keep]
        chs = [chunks[i] for i in keep]
        self.document_id.extend(ids)
        self.chunk.extend(chs)
        self.metadata.extend(metadata[i] for i in keep)
        enc_d = [_avro_nullable_string(d) for d in ids]
        enc_c = [_avro_nullable_string(c) for c in chs]
        self.avro_document_id.extend(enc_d)
        self.avro_chunk.extend(enc_c)
        self.arena_document_id.extend(enc_d)
        self.arena_chunk.extend(enc_c)
        for j, d in enumerate(ids):
            if d is not None:
                self._row_of[d] = first + j

    def load_columns(self, document_ids, chunks, metadata=None) -> None:
        """Attach the non-vector columns for rows whose vectors are ALREADY in the index (bulk load of a pre-built
        shard): row i of the index gets document_ids[i] / chunks[i]."""
        assert len(self.document_id) == 0 and len(document_ids) == len(chunks)
        metadata = metadata or [{} for _ in range(len(document_ids))]
        if self.filter_schema is not None and len(metadata):
            self.index.set_tags(np.arange(len(metadata)), self.filter_schema.tags(metadata))
        for d, c, m in zip(document_ids, chunks, metadata):
            if d is not None:
                self._row_of[d] = len(self.document_id)
            self.document_id.append(d)
            self.chunk.append(c)
            self.metadata.append(m)
            self._push_avro(d, c)

    def save(self, directory: str, source_offsets: dict[str, int] | None = None) -> int:
        """Checkpoint: the index snapshot (if the index supports it), the side table as JSON lines, and LAST a manifest
        naming both (generation-numbered files, each written to a temporary name and renamed), so a crash at any point
        leaves the previous checkpoint intact and readable.  ``source_offsets`` ({"<topic>-<partition>": next offset})
        records how far into its source topic the table's content reaches: a resumed sink continues exactly there."""
        import json
        import os
        os.makedirs(directory, exist_ok=True)
        prev = self._read_manifest(directory)
        gen = (prev["generation"] + 1) if prev else 1
        n = len(self)
        files = {"columns": f"columns.{gen}.jsonl"}
        if hasattr(self.index, "snapshot"):
            files["index"] = f"index.{gen}.npz"
            self.index.snapshot(os.path.join(directory, files["index"]))          # atomic (tmp + rename) in the index
        tmp = os.path.join(directory, files["columns"] + ".tmp")
        with open(tmp, "w", encoding="utf-8") as f:
            for d, c, m in zip(self.document_id, self.chunk, self.metadata):
                f.write(json.dumps({"document_id": d, "chunk": c, "metadata": m}, ensure_ascii=False) + "\n")
            f.flush()
            os.fsync(f.fileno())
        os.replace(tmp, os.path.join(directory, files["columns"]))
        man = {"generation": gen, "rows": n, "files": files, "source_offsets": source_offsets or {},
               "similarity": self.similarity, "filter_fields": list(self.filter_fields),
               "filter_bits": self.filter_schema.to_json()["bits"] if self.filter_schema is not None else []}
        tmp = os.path.join(directory, "manifest.json.tmp")
        with open(tmp, "w") as f:
            json.dump(man, f)
            f.flush()
            os.fsync(f.fileno())
        os.replace(tmp, os.path.join(directory, "manifest.json"))
        if prev:                                                                  # the old generation is garbage now
            for name in prev["files"].values():
                try:
                    os.remove(os.path.join(directory, name))
                except OSError:
                    pass
        return n

    @staticmethod
    def _read_manifest(directory: str):
        import json
        import os
        try:
            with open(os.path.join(directory, "manifest.json")) as f:
                return json.load(f)
        except (OSError, ValueError):
            return None

    @classmethod
    def has_checkpoint(cls, directory: str) -> bool:
        return cls._read_manifest(directory) is not None

    def load(self, directory: str) -> int:
        """Resume from ``save``: restores the index, the side table and ``source_offsets`` (call on an empty table).
        A checkpoint taken under another similarity is refused (a manifest that does not name one is a cosine one), as
        is one taken with other filter fields; a checkpoint that predates filter fields rebuilds the tags from its
        metadata column."""
        import json
        import os
        assert len(self) == 0, "load() needs an empty table"
        man = self._read_manifest(directory)
        if man is None:
            raise FileNotFoundError(f"no checkpoint manifest in {directory}")
        rows = []
        with open(os.path.join(directory, man["files"]["columns"]), encoding="utf-8") as f:
            for line in f:
                rows.append(json.loads(line))
        saved = man.get("similarity", "cosine")
        if saved != self.similarity:
            raise ValueError(f"checkpoint in {directory} was taken with similarity {saved!r}; this table's index uses "
                             f"{self.similarity!r}: rankings and row terms differ, rebuild the table from the log instead")
        saved_fields = man.get("filter_fields")
        if saved_fields is not None and tuple(saved_fields) != self.filter_fields:
            raise ValueError(f"checkpoint in {directory} was taken with filter fields {list(saved_fields)}; this table "
                             f"declares {list(self.filter_fields)}: rebuild the table from the log instead")
        if len(rows) != man["rows"]:
            raise ValueError(f"snapshot mismatch: manifest says {man['rows']} rows, columns file has {len(rows)}")
        if self.filter_schema is not None and saved_fields is not None:
            # the saved bit dictionary: the tags recomputed below are the ones the checkpoint's filters were built on
            self.filter_schema = FilterSchema.from_json({"fields": saved_fields, "bits": man.get("filter_bits", [])})
        if hasattr(self.index, "restore") and "index" in man["files"]:
            n = self.index.restore(os.path.join(directory, man["files"]["index"]))
            if n != len(rows):
                raise ValueError(f"snapshot mismatch: {n} vectors, {len(rows)} column rows")
        self.load_columns([r["document_id"] for r in rows], [r["chunk"] for r in rows], [r["metadata"] for r in rows])
        # a re-published document tombstones its old row: the live row of an id is its LAST occurrence
        self.source_offsets = dict(man.get("source_offsets") or {})
        return len(self)

    def clear(self) -> None:
        """What scripts/common/clear_mongodb.py:98-158 does before a re-publish."""
        self.index.reset()
        if self.filter_schema is not None:
            self.filter_schema = FilterSchema(self.filter_fields)
        self.document_id.clear()
        self.chunk.clear()
        self.metadata.clear()
        self._row_of.clear()
        self.avro_document_id.clear()
        self.avro_chunk.clear()
        self.arena_document_id.clear()
        self.arena_chunk.clear()


def index_similarity(index) -> str:
    return getattr(index, "similarity", "cosine")


def atlas_score(score: float, similarity: str = "cosine") -> float:
    """The score MongoDB Atlas Vector Search reports for a raw engine score, as Atlas's documentation states the
    normalisation (restated from there, not from the reference tree): cosine and dotProduct map to [0, 1] as
    (1 + s) / 2, euclidean distance d as 1 / (1 + d).  The engine's native score is the raw value (what BASELINE.json's
    numpy yardstick uses).  Apply this where a downstream consumer expects Atlas's."""
    if similarity == "euclidean":
        return 1.0 / (1.0 + score)
    if similarity in ("cosine", "dotProduct"):
        return 0.5 * (1.0 + score)
    raise ValueError(f"unknown similarity {similarity!r}")


def wire_score_mode(score_mode: str, similarity: str) -> int:
    """score_mode argument of sa_wire_encode_search_results: 0 raw, 1 (1 + s) / 2, 2 1 / (1 + d)."""
    if score_mode != "atlas":
        return 0
    return 2 if similarity == "euclidean" else 1


def vector_search_agg(table: VectorTable, descriptor: str, query_vectors: np.ndarray, k: int,
                      score_mode: str = "cosine", filter=None) -> list[list[SearchHit]]:
    """VECTOR_SEARCH_AGG(table, DESCRIPTOR(descriptor), query_vector, k) for a batch of query vectors; k <= the index's
    max_k (at most 64, Atlas's ``limit``), each query's hits exact and best first.
    ``score_mode``: "cosine" (the raw value of the index's similarity, default) or "atlas" (``atlas_score``).
    ``filter``: an MQL document over the table's filter fields (``filters.compile_filter``), or a list with one per
    query; each query's top-k is then the exact top-k of the rows its filter matches."""
    if score_mode not in ("cosine", "atlas"):
        raise ValueError("score_mode must be 'cosine' or 'atlas'")
    if descriptor != table.embedding_column:
        raise ValueError(f"table {table.name} has no vector column {descriptor!r}")
    q = np.ascontiguousarray(query_vectors, dtype=np.float32)
    if q.ndim == 1:
        q = q[None, :]
    if q.shape[0] == 0:
        return []
    if filter is None:
        score, idx = table.index.search_host(q, k)
    else:
        if table.filter_schema is None:
            raise ValueError(f"table {table.name} declares no filter fields")
        docs = filter if isinstance(filter, (list, tuple)) else [filter] * q.shape[0]
        if len(docs) != q.shape[0]:
            raise ValueError(f"{len(docs)} filters for {q.shape[0]} queries")
        f = np.stack([compile_filter(table.filter_schema, d) for d in docs])
        score, idx = table.index.search_host(q, k, filters=f)
    out = []
    for r in range(q.shape[0]):
        hits = []
        for s, i in zip(score[r].tolist(), idx[r].tolist()):
            if i < 0:
                break
            s = atlas_score(s, table.similarity) if score_mode == "atlas" else s
            hits.append(SearchHit(table.document_id[i], table.chunk[i], float(s), int(i), table.metadata[i]))
        out.append(hits)
    return out


def search_results_avro_body(table: VectorTable, query: str | None, score_row, idx_row, n: int = 3,
                             score_mode: str = "cosine") -> bytes:
    """Avro body of one ``search_results`` record straight from a result row (scores, table rows) -- byte-identical to
    encoding ``flatten_search_results(...)`` with the generic codec, without building the dict."""
    import struct
    parts = [_avro_nullable_string(query)]
    for j in range(n):
        i = int(idx_row[j]) if j < len(idx_row) else -1
        if i < 0:
            parts.append(b"\x00\x00\x00")  # document_id, chunk, score all null
        else:
            parts.append(table.avro_document_id[i])
            parts.append(table.avro_chunk[i])
            sc = float(score_row[j])
            parts.append(b"\x02" + struct.pack("<d", atlas_score(sc, table.similarity) if score_mode == "atlas" else sc))
    return b"".join(parts)


def flatten_search_results(query: str | None, hits: list[SearchHit], n: int = 3) -> dict:
    """The projection of main.tf:292: query + document_id_i / chunk_i / score_i for i = 1..n (null-padded)."""
    rec = {"query": query}
    for i in range(1, n + 1):
        h = hits[i - 1] if i <= len(hits) else None
        rec[f"document_id_{i}"] = h.document_id if h else None
        rec[f"chunk_{i}"] = h.chunk if h else None
        rec[f"score_{i}"] = h.score if h else None
    return rec


def project_search_results(hits: list[SearchHit], columns: dict[str, str], n: int = 3) -> dict:
    """Generic form of the projection for tables with metadata columns, e.g. Lab4's
    ``vs.search_results[i].chunk AS policy_chunk_i, ... .pages AS policy_pages_i, ...`` (LAB4-Walkthrough.md:280-300):
    ``columns`` maps a table column (document_id, chunk, score or a metadata column) to its output prefix."""
    rec = {}
    for i in range(1, n + 1):
        h = hits[i - 1] if i <= len(hits) else None
        for col, prefix in columns.items():
            if h is None:
                v = None
            elif col in ("document_id", "chunk", "score"):
                v = getattr(h, col)
            else:
                v = h.metadata.get(col)
            rec[f"{prefix}_{i}"] = v
    return rec


def rag_prompt(rec: dict) -> str:
    """The CONCAT(...) of main.tf:331, character for character (SQL '' -> ', \\n -> newline)."""
    def s(v):
        return "" if v is None else str(v)
    return (
        "Based on the following search results, provide a helpful and comprehensive response to the user query "
        "based upon the relevant retrieved documents. Cite the exact parts of the retrieved documents whenever "
        "possible.\n\nUSER QUERY: " + s(rec["query"]) + "\n\nSEARCH RESULTS:\n\n"
        "Document 1 (Similarity Score: " + s(rec["score_1"]) + "):\nSource: " + s(rec["document_id_1"]) +
        "\nContent: " + s(rec["chunk_1"]) +
        "\n\nDocument 2 (Similarity Score: " + s(rec["score_2"]) + "):\nSource: " + s(rec["document_id_2"]) +
        "\nContent: " + s(rec["chunk_2"]) +
        "\n\nDocument 3 (Similarity Score: " + s(rec["score_3"]) + "):\nSource: " + s(rec["document_id_3"]) +
        "\nContent: " + s(rec["chunk_3"]) +
        "\n\nINSTRUCTIONS:\n- Synthesize information from the most relevant documents above\n"
        "- Provide specific, actionable guidance when possible\n- Reference document sources in your response\n"
        "- If the search results don't contain relevant information, say so clearly\n\nRESPONSE:")
