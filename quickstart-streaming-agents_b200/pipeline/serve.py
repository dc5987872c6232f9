"""Local serve loop for the Lab2 RAG pipeline.

What Confluent Cloud Flink runs as continuous statements, this process runs as consumer/producer stages over
topics with the same names and Avro schemas (SURVEY.md section 8b):

  documents        --embed(stub)-->  documents_embed  --sink-->  VectorTable (HBM)         LAB2-Walkthrough.md:41-51
  queries          --embed(stub)-->  queries_embed                                          main.tf:253
  queries_embed    --VECTOR_SEARCH_AGG(table, DESCRIPTOR(embedding), embedding, k)-->  search_results   main.tf:292
  search_results   --RAG prompt + generator(stub)-->  search_results_response              main.tf:331

Records on ``queries_embed`` / ``documents_embed`` may also come from outside (pre-computed embeddings).
Delivery is at-least-once: each stage commits its consumer offsets after its outputs are flushed.
A poison record (bad magic byte, truncated Avro, wrong embedding length) is quarantined to ``<topic>.dlq``
with the error text in its key, and the stage moves on.

Durability.  The reference's vector table lives in Atlas and survives a restart of the Flink statements; here it lives
in HBM and does not.  So the sink stage's read position is tied to the TABLE's state, never to a consumer group's
committed offsets: a table restored from a checkpoint resumes ``documents_embed`` at the offsets stored inside that
checkpoint, and a table that starts empty re-reads ``documents_embed`` from its low watermark (the durable log rebuilds
it).  Every other stage resumes from its group offsets as usual.

Search stage.  The hot loop works a batch at a time with no per-record Python objects: one read of the partition log
(``consume_raw``), native split + Avro decode of the batch straight into a page-locked buffer (``sa_wire_*``), the
two-slot host search of the C ABI, native Avro encode + log framing of the results, one append.  Records in an unusual
shape fall back to the generic codec, record by record, inside the same batch (order is preserved).
"""
from __future__ import annotations

import ctypes as C
import json
import logging
import struct
import time

import numpy as np

from ..embed.stub import StubEmbedder
from ..operator import VectorTable, rag_prompt, search_results_avro_body, wire_score_mode
from ..transport.filelog import Message
from ..wire import avro, schemas
from ..wire.registry import SchemaRegistry

log = logging.getLogger(__name__)


def stub_generator(prompt: str, rec: dict) -> str:
    """Stand-in for ml_predict('llm_textgen_model', prompt) (main.tf:331): a deterministic extractive answer that
    cites the retrieved sources, so the test shape "response is non-empty" (testing/e2e/test_lab2.py:112-135) and
    a human reading the topic both get something sensible."""
    parts = []
    for i in (1, 2, 3):
        if rec.get(f"document_id_{i}") is not None:
            chunk = (rec.get(f"chunk_{i}") or "").strip().replace("\n", " ")
            parts.append(f"[{rec[f'document_id_{i}']}] (score {rec[f'score_{i}']:.4f}): {chunk[:240]}")
    if not parts:
        return "The search results don't contain relevant information for this query."
    return "Based on the retrieved documents:\n" + "\n".join(parts)


class Codec:
    """Avro + Confluent framing for one log directory (schema ids from the registry stub, compiled codecs)."""

    def __init__(self, log_dir: str):
        self.registry = SchemaRegistry(log_dir)
        self._enc: dict[str, tuple[bytes, avro.CompiledSchema]] = {}
        self._dec: dict[int, avro.CompiledSchema] = {}

    def schema_id(self, topic: str) -> int:
        return struct.unpack(">I", self._encoder(topic)[0][1:5])[0]

    def _encoder(self, topic: str):
        e = self._enc.get(topic)
        if e is None:
            sid = self.registry.register(f"{topic}-value", schemas.TOPIC_SCHEMAS[topic])
            e = self._enc[topic] = (avro.frame(sid, b""), avro.CompiledSchema(schemas.TOPIC_SCHEMAS[topic]))
        return e

    def header(self, topic: str) -> bytes:
        return self._encoder(topic)[0]

    def encode(self, topic: str, record: dict) -> bytes:
        header, cs = self._encoder(topic)
        return cs.encode(record, prefix=header)

    def decode(self, raw: bytes) -> dict:
        if len(raw) < 5:
            raise avro.AvroError(f"Avro payload too short ({len(raw)} bytes)")
        if raw[0] != avro.MAGIC:
            raise avro.AvroError(f"Invalid Avro magic byte: {raw[0]}")
        sid = struct.unpack_from(">I", raw, 1)[0]
        cs = self._dec.get(sid)
        if cs is None:
            cs = self._dec[sid] = avro.CompiledSchema(self.registry.get(sid))
        return cs.decode(raw, 5)


class Lab2Pipeline:
    def __init__(self, log_dir: str, table: VectorTable, embedder=None, k: int = 3, max_batch: int = 1024,
                 group: str = "sa-lab2", generator=stub_generator, score_mode: str = "cosine", native: bool | None = None,
                 metrics_file: str | None = None, metrics_every_s: float = 5.0, transport=None, client_conf: dict | None = None):
        """``transport``: a module with ``Producer`` / ``Consumer`` / ``TopicPartition`` -- ``transport.filelog`` (default,
        topics are files under ``log_dir``) or ``transport.kafka`` (a real cluster through confluent_kafka; ``client_conf``
        carries bootstrap.servers etc., ``log_dir`` then only holds the schema-registry stub)."""
        if score_mode not in ("cosine", "atlas"):
            raise ValueError("score_mode must be 'cosine' (the raw score of the index's similarity) or 'atlas' (what "
                             "MongoDB Atlas reports: (1 + s) / 2, or 1 / (1 + d) for euclidean)")
        self.log_dir = log_dir
        self.table = table
        self.embedder = embedder or StubEmbedder(table.index.dim)
        self.k = k
        self.max_batch = max_batch
        self.generator = generator
        self.score_mode = score_mode
        self.codec = Codec(log_dir)
        tp_mod = transport
        if tp_mod is None:
            from ..transport import filelog as tp_mod
        TopicPartition = tp_mod.TopicPartition
        base = dict(client_conf or {})
        base["log.dir"] = log_dir
        self.producer = tp_mod.Producer(base)
        conf = dict(base, **{"group.id": group, "auto.offset.reset": "earliest", "enable.auto.commit": False})
        self.consumers = {}
        for t in ("documents", "documents_embed", "queries", "queries_embed", "search_results"):
            c = tp_mod.Consumer(conf)
            c.subscribe([t])
            self.consumers[t] = c
        # the sink reads from where the TABLE's content ends, not from where some earlier process committed
        sink = self.consumers["documents_embed"]
        if table.source_offsets:
            sink.seek_to_beginning("documents_embed")      # partitions the checkpoint has never seen start at their beginning
            for key, off in table.source_offsets.items():
                t, _, p = key.rpartition("-")
                if t == "documents_embed":
                    sink.seek(TopicPartition(t, int(p), int(off)))
        else:
            sink.seek_to_beginning("documents_embed")
        self.stats = {"documents": 0, "queries": 0, "searches": 0, "responses": 0, "quarantined": 0,
                      "search_seconds": 0.0, "search_batches": 0, "snapshots": 0}
        # native batch codecs (include/sa_wire.h); the generic Python codec stays the reference implementation
        self._wire = None
        if native is None or native:
            try:
                from .. import capi
                self._wire = capi.load()
            except Exception:
                if native:
                    raise
        self._qbuf = None          # two query staging buffers (page-locked when the index can DMA from them)
        self._rbuf = [None, None]  # two reusable read buffers for the partition-log slices of the native search stage
        self._lat_ms: list[float] = []
        self._metrics_file, self._metrics_every_s = metrics_file, metrics_every_s
        self._metrics_t0 = time.time()
        self._metrics_q0 = 0
        self._sink_dirty = False
        # further statements over the same table, run at the end of every pass (pipeline/lateral.py: the Lab3 / Lab4
        # form of the operator, joined LATERALly onto an upstream stream)
        self.extra_stages: list = []

    # ------------------------------------------------------------------ helpers
    def _decode_all(self, topic: str, msgs):
        good = []
        for m in msgs:
            try:
                good.append((m, self.codec.decode(m.value())))
            except Exception as e:  # poison message: quarantine, keep going
                self.stats["quarantined"] += 1
                log.warning("quarantined %s[%d]@%d: %s", topic, m.partition(), m.offset(), e)
                self.producer.produce(f"{topic}.dlq", key=str(e), value=m.value())
        return good

    def _drain(self, topic: str):
        c = self.consumers[topic]
        msgs = c.consume(self.max_batch, 0.0)
        return c, msgs, self._decode_all(topic, msgs)

    def _check_vec(self, topic, m, vec):
        dim = self.table.index.dim
        if vec is None or len(vec) != dim or not np.isfinite(vec).all():
            self.stats["quarantined"] += 1
            why = f"embedding must be {dim} finite floats"
            log.warning("quarantined %s@%d: %s", topic, m.offset(), why)
            self.producer.produce(f"{topic}.dlq", key=why, value=m.value())
            return False
        return True

    # ------------------------------------------------------------------ stages
    def stage_documents(self) -> int:
        c, msgs, recs = self._drain("documents")
        for m, r in recs:
            text = r.get("document_text") or ""
            vec = self.embedder.embed(text)
            out = {"document_id": r.get("document_id"), "chunk": text, "embedding": vec}
            out.update({c: r.get(c) for c in schemas.METADATA_COLUMNS})   # Lab4-style metadata passthrough
            self.producer.produce("documents_embed", key=m.key(), value=self.codec.encode("documents_embed", out))
        if msgs:
            self.producer.flush()
            c.commit()
        return len(msgs)

    def stage_sink(self) -> int:
        """documents_embed -> vector table.  Batch path: one read of the partition log, native split + decode of ids, chunks
        and embeddings (sa_wire_decode_documents_embed; the six metadata columns are validated natively and decoded only
        when they are not all null), one upsert per batch; records in an unusual shape go through the generic codec."""
        c = self.consumers["documents_embed"]
        if self._wire is not None and hasattr(c, "consume_raw"):
            return self._stage_sink_native()
        return self._stage_sink_generic()

    def _stage_sink_native(self) -> int:
        c = self.consumers["documents_embed"]
        lib, dim = self._wire, self.table.index.dim
        if not hasattr(self, "_meta_codec"):
            fields = [f for f in schemas.DOCUMENTS_EMBED_VALUE["fields"] if f["name"] in schemas.METADATA_COLUMNS]
            self._meta_codec = avro.CompiledSchema({"type": "record", "name": "documents_embed_metadata", "fields": fields})
            self._null_meta = {col: None for col in schemas.METADATA_COLUMNS}
        total = 0
        while True:
            raw = c.consume_raw(self.max_batch)
            if raw is None:
                break
            topic, part, first, n, data = raw
            total += n
            voff, vlen = np.empty(n, np.uint64), np.empty(n, np.uint32)
            if lib.sa_wire_split_log(data, len(data), n, voff.ctypes.data, vlen.ctypes.data, None, None, None):
                raise avro.AvroError("corrupt log slice: " + lib.sa_last_error().decode())
            vecs = np.empty((n, dim), np.float32)
            io, co, mo = (np.empty(n, np.uint64) for _ in range(3))
            il, cl, ml = (np.empty(n, np.uint32) for _ in range(3))
            status = np.empty(n, np.uint8)
            n_ok = C.c_int()
            if lib.sa_wire_decode_documents_embed(data, voff.ctypes.data, vlen.ctypes.data, n, dim,
                                                  self.codec.schema_id("documents_embed"), vecs.ctypes.data, io.ctypes.data,
                                                  il.ctypes.data, co.ctypes.data, cl.ctypes.data, mo.ctypes.data,
                                                  ml.ctypes.data, status.ctypes.data, C.byref(n_ok)):
                raise avro.AvroError(lib.sa_last_error().decode())
            ids, chunks, metas, keep = [], [], [], []
            io_l, il_l, co_l, cl_l, mo_l, ml_l, st_l = (x.tolist() for x in (io, il, co, cl, mo, ml, status))
            for i in range(n):
                if st_l[i] == 0:
                    ids.append(None if il_l[i] == 0xFFFFFFFF else data[io_l[i]:io_l[i] + il_l[i]].decode("utf-8"))
                    chunks.append(None if cl_l[i] == 0xFFFFFFFF else data[co_l[i]:co_l[i] + cl_l[i]].decode("utf-8"))
                    mb = data[mo_l[i]:mo_l[i] + ml_l[i]]
                    metas.append(dict(self._null_meta) if mb == b"\x00\x00\x00\x00\x00\x00" else self._meta_codec.decode(mb))
                    keep.append(i)
                    continue
                value = None if vlen[i] == 0xFFFFFFFF else data[int(voff[i]):int(voff[i]) + int(vlen[i])]
                m = Message(topic, part, first + i, None, value, 0)
                got = self._decode_all("documents_embed", [m])
                if not got or not self._check_vec("documents_embed", m, got[0][1].get("embedding")):
                    continue
                r = got[0][1]
                vecs[i] = r["embedding"]
                ids.append(r.get("document_id"))
                chunks.append(r.get("chunk"))
                metas.append({col: r.get(col) for col in schemas.METADATA_COLUMNS})
                keep.append(i)
            if ids:
                self.table.upsert_many(ids, chunks, vecs if len(keep) == n else vecs[keep], metas)
                self.stats["documents"] += len(ids)
                self._sink_dirty = True
            self.producer.flush()     # quarantined records, if any
            c.commit_upto(topic, part, first + n)   # informational only: the sink's start position comes from the table
        return total

    def _stage_sink_generic(self) -> int:
        c, msgs, recs = self._drain("documents_embed")
        ids, chunks, vecs, metas = [], [], [], []
        for m, r in recs:
            vec = r.get("embedding")
            if not self._check_vec("documents_embed", m, vec):
                continue
            ids.append(r.get("document_id"))
            chunks.append(r.get("chunk"))
            vecs.append(vec)
            metas.append({c: r.get(c) for c in schemas.METADATA_COLUMNS})
        if ids:
            self.table.upsert_many(ids, chunks, np.stack(vecs), metas)
            self.stats["documents"] += len(ids)
            self._sink_dirty = True
        if msgs:
            self.producer.flush()
            c.commit()      # informational only: the sink's start position comes from the table (see module docstring)
        return len(msgs)

    def stage_queries(self) -> int:
        c, msgs, recs = self._drain("queries")
        for m, r in recs:
            q = r.get("query") or ""
            self.producer.produce("queries_embed", value=self.codec.encode(
                "queries_embed", {"query": q, "embedding": self.embedder.embed(q)}))
        if msgs:
            self.stats["queries"] += len(recs)
            self.producer.flush()
            c.commit()
        return len(msgs)

    def _decode_queries_embed_fast(self, msgs):
        """Batch decode of `queries_embed` records in their usual shape -- non-null query string, non-null single-block
        array of dim non-null floats -- with one strided numpy gather for all embeddings.  Returns (texts, vectors,
        leftovers): messages in any other shape are returned in `leftovers` for the generic per-record path."""
        dim = self.table.index.dim
        sid = self.codec.schema_id("queries_embed")
        header = bytes([0]) + struct.pack(">I", sid)
        block = bytearray()
        avro.write_long(block, dim)
        block = bytes(block)
        span = 5 * dim
        texts, views, leftovers = [], [], []
        for m in msgs:
            raw = m.value()
            try:
                if raw[:5] != header or raw[5] != 2:
                    raise ValueError
                n, pos = avro.read_long(raw, 6)
                end = pos + n
                if raw[end] != 2 or raw[end + 1:end + 1 + len(block)] != block:
                    raise ValueError
                off = end + 1 + len(block)
                if len(raw) != off + span + 1 or raw[-1] != 0:
                    raise ValueError
                text = raw[pos:end].decode("utf-8")
            except (ValueError, IndexError, TypeError):
                leftovers.append(m)
                continue
            texts.append(text)
            views.append(np.frombuffer(raw, dtype=np.uint8, count=span, offset=off))
        if not views:
            return [], np.empty((0, dim), np.float32), leftovers
        flat = np.stack(views).reshape(len(views), dim, 5)
        ok = (flat[:, :, 0] == 2).all(axis=1)
        vecs = np.ascontiguousarray(flat[:, :, 1:]).view("<f4").reshape(len(views), dim)
        ok &= np.isfinite(vecs).all(axis=1)
        if not ok.all():  # a null / non-finite item somewhere: let the generic path judge those records
            bad = set(np.flatnonzero(~ok).tolist())
            fast_msgs = [m for m in msgs if m not in leftovers]
            leftovers.extend(fast_msgs[i] for i in sorted(bad))
            keep = [i for i in range(len(views)) if i not in bad]
            texts = [texts[i] for i in keep]
            vecs = vecs[keep]
        return texts, vecs, leftovers

    def _decode_batch(self, msgs):
        """queries_embed messages -> (texts, vectors) in stream order: fast batch path, generic codec (and quarantine) for
        the records the fast path does not take."""
        texts, vecs, leftovers = self._decode_queries_embed_fast(msgs)
        if not leftovers:
            return texts, np.ascontiguousarray(vecs, dtype=np.float32)
        left = {id(m) for m in leftovers}
        fast_iter = iter(range(len(texts)))
        out_t, out_v = [], []
        for m in msgs:
            if id(m) not in left:
                i = next(fast_iter)
                out_t.append(texts[i])
                out_v.append(vecs[i])
                continue
            got = self._decode_all("queries_embed", [m])
            if got and self._check_vec("queries_embed", m, got[0][1].get("embedding")):
                out_t.append(got[0][1].get("query"))
                out_v.append(np.asarray(got[0][1]["embedding"], dtype=np.float32))
        dim = self.table.index.dim
        return out_t, (np.ascontiguousarray(np.stack(out_v), dtype=np.float32) if out_v else np.empty((0, dim), np.float32))

    def _emit_results(self, texts, score, idx) -> None:
        header = self.codec.header("search_results")
        n_out = schemas.RESULTS_PER_QUERY
        for r, q in enumerate(texts):
            self.producer.produce("search_results", value=header + search_results_avro_body(
                self.table, q, score[r], idx[r], n_out, self.score_mode))
        self.stats["searches"] += len(texts)

    # ---- native batch path -------------------------------------------------------------------------------------------
    def _query_buffers(self):
        if self._qbuf is None:
            dim = self.table.index.dim
            try:        # page-locked: the engine DMAs straight from the decode buffer
                from ..engine import pinned_array
                self._qbuf = [pinned_array((self.max_batch, dim), np.float32) for _ in range(2)]
            except Exception:
                self._qbuf = [np.empty((self.max_batch, dim), np.float32) for _ in range(2)]
        return self._qbuf

    def _decode_raw_batch(self, raw, slot):
        """One partition slice -> (n_good, vectors view, text buffer, text_off, text_len).  Fast shape natively; anything
        else through the generic codec (which also quarantines), in place, so the batch keeps its order."""
        topic, part, first, n, data = raw
        lib, dim = self._wire, self.table.index.dim
        data = np.frombuffer(data, np.uint8)       # bytes, or a view of the reusable read buffer: no copy either way
        dptr = data.ctypes.data
        voff = np.empty(n, np.uint64)
        vlen = np.empty(n, np.uint32)
        rc = lib.sa_wire_split_log(dptr, len(data), n, voff.ctypes.data, vlen.ctypes.data, None, None, None)
        if rc:
            raise avro.AvroError("corrupt log slice: " + lib.sa_last_error().decode())
        vecs = self._query_buffers()[slot]
        toff = np.empty(n, np.uint64)
        tlen = np.empty(n, np.uint32)
        status = np.empty(n, np.uint8)
        n_ok = C.c_int()
        rc = lib.sa_wire_decode_queries_embed(dptr, voff.ctypes.data, vlen.ctypes.data, n, dim,
                                              self.codec.schema_id("queries_embed"), vecs.ctypes.data, toff.ctypes.data,
                                              tlen.ctypes.data, status.ctypes.data, C.byref(n_ok))
        if rc:
            raise avro.AvroError(lib.sa_last_error().decode())
        text_buf = data
        if n_ok.value != n:
            extra = bytearray()
            keep = np.ones(n, bool)
            for i in np.flatnonzero(status).tolist():
                value = None if vlen[i] == 0xFFFFFFFF else data[int(voff[i]):int(voff[i]) + int(vlen[i])].tobytes()
                m = Message(topic, part, first + i, None, value, 0)
                got = self._decode_all("queries_embed", [m])
                vec = got[0][1].get("embedding") if got else None
                if not got or not self._check_vec("queries_embed", m, vec):
                    keep[i] = False
                    continue
                vecs[i] = vec
                q = got[0][1].get("query")
                if q is None:
                    tlen[i] = 0xFFFFFFFF
                else:
                    qb = q.encode("utf-8")
                    toff[i] = len(data) + len(extra)
                    tlen[i] = len(qb)
                    extra += qb
            if extra:
                text_buf = np.frombuffer(data.tobytes() + bytes(extra), np.uint8)
            if not keep.all():
                good = np.flatnonzero(keep)
                vecs[:len(good)] = vecs[good]
                toff, tlen = toff[good], tlen[good]
                n = len(good)
        return n, vecs[:n], text_buf, toff, tlen

    def _emit_results_native(self, n, text_buf, toff, tlen, score, idx) -> None:
        lib, t = self._wire, self.table
        rows = np.ascontiguousarray(idx, dtype=np.int64)
        score = np.ascontiguousarray(score, dtype=np.float32)
        k = score.shape[1]
        rec_off = np.empty(n + 1, np.uint64)
        need = C.c_uint64()
        args = (n, k, schemas.RESULTS_PER_QUERY, self.codec.schema_id("search_results"), text_buf.ctypes.data, toff.ctypes.data,
                tlen.ctypes.data, score.ctypes.data, rows.ctypes.data, t.arena_document_id.data.ctypes.data,
                t.arena_document_id.off.ctypes.data, t.arena_chunk.data.ctypes.data, t.arena_chunk.off.ctypes.data, len(t),
                wire_score_mode(self.score_mode, t.similarity), int(time.time() * 1000))
        lib.sa_wire_encode_search_results(*args, None, 0, rec_off.ctypes.data, C.byref(need))   # sizing pass
        out = np.empty(int(need.value), np.uint8)
        rc = lib.sa_wire_encode_search_results(*args, out.ctypes.data, out.size, rec_off.ctypes.data, C.byref(need))
        if rc:
            raise avro.AvroError(lib.sa_last_error().decode())
        self.producer.produce_framed("search_results", out.data, rec_off[:n])
        self.stats["searches"] += n

    def _note_latency(self, t_submit, n):
        self._lat_ms.append((time.perf_counter() - t_submit) * 1e3)
        self.stats["search_batches"] += 1
        if self._metrics_file and time.time() - self._metrics_t0 >= self._metrics_every_s:
            self.write_metrics()

    def write_metrics(self) -> dict:
        """One JSON line of batch-latency percentiles (consume -> results flushed) and throughput since the last line."""
        now = time.time()
        lat = np.asarray(self._lat_ms or [0.0])
        row = {"ts": now, "batches": len(self._lat_ms), "queries": self.stats["searches"] - self._metrics_q0,
               "qps": (self.stats["searches"] - self._metrics_q0) / max(now - self._metrics_t0, 1e-9),
               "batch_latency_ms": {"p50": float(np.percentile(lat, 50)), "p99": float(np.percentile(lat, 99)),
                                    "max": float(lat.max())}, "table_rows": len(self.table)}
        if self._metrics_file:
            with open(self._metrics_file, "a") as f:
                f.write(json.dumps(row) + "\n")
        self._lat_ms, self._metrics_t0, self._metrics_q0 = [], now, self.stats["searches"]
        return row

    def stage_search(self) -> int:
        """queries_embed -> VECTOR_SEARCH_AGG -> search_results.  When the index offers the split host call
        (``search_host_submit`` / ``search_host_wait``), batches are software-pipelined: batch i+1 is read and decoded
        while the GPU searches batch i.  Offsets of a batch are committed only after its results are flushed."""
        if (self._wire is not None and len(self.table) == self.table.arena_document_id.n
                and hasattr(self.consumers["queries_embed"], "consume_raw")):
            return self._stage_search_native()
        return self._stage_search_generic()

    def _stage_search_native(self) -> int:
        c = self.consumers["queries_embed"]
        index = self.table.index
        pipelined = hasattr(index, "search_host_submit")
        total, slot, pending = 0, 0, None
        while True:
            raw = c.consume_raw(self.max_batch, self._rbuf[slot])
            batch = None
            if raw is not None:
                if self._rbuf[slot] is None or len(raw[4]) > len(self._rbuf[slot]):   # size the buffer to the slices seen
                    self._rbuf[slot] = np.empty(len(raw[4]) + len(raw[4]) // 8 + 4096, np.uint8)
                total += raw[3]
                t_in = time.perf_counter()
                n, vecs, text_buf, toff, tlen = self._decode_raw_batch(raw, slot)
                batch = (raw, n, vecs, text_buf, toff, tlen, t_in)
                if n and pipelined:
                    t0 = time.perf_counter()
                    index.search_host_submit(vecs, self.k, slot)
                    self.stats["search_seconds"] += time.perf_counter() - t0
            if pending is not None:      # collect the previous batch while the new one runs
                (p_raw, p_n, _, p_text, p_toff, p_tlen, p_t), p_slot = pending
                t0 = time.perf_counter()
                score, idx = index.search_host_wait(p_slot)
                self.stats["search_seconds"] += time.perf_counter() - t0
                self._emit_results_native(p_n, p_text, p_toff, p_tlen, score, idx)
                c.commit_upto(p_raw[0], p_raw[1], p_raw[2] + p_raw[3])
                self._note_latency(p_t, p_n)
                pending = None
            if batch is None:
                break
            raw, n, vecs, text_buf, toff, tlen, t_in = batch
            if n and pipelined:
                pending = (batch, slot)
                slot ^= 1
            else:
                if n:
                    t0 = time.perf_counter()
                    score, idx = index.search_host(vecs, self.k)
                    self.stats["search_seconds"] += time.perf_counter() - t0
                    self._emit_results_native(n, text_buf, toff, tlen, score, idx)
                    self._note_latency(t_in, n)
                self.producer.flush()  # carries any quarantined records of this batch
                c.commit_upto(raw[0], raw[1], raw[2] + raw[3])
        return total

    def _stage_search_generic(self) -> int:
        c = self.consumers["queries_embed"]
        index = self.table.index
        pipelined = hasattr(index, "search_host_submit")
        total = 0
        pending = None  # (messages, texts, slot) of the batch the GPU is working on
        slot = 0
        while True:
            msgs = c.consume(self.max_batch, 0.0)
            batch = None
            if msgs:
                total += len(msgs)
                texts, vecs = self._decode_batch(msgs)
                batch = (msgs, texts, vecs)
            if batch is not None and len(batch[1]) and pipelined:
                t0 = time.perf_counter()
                index.search_host_submit(batch[2], self.k, slot)
                self.stats["search_seconds"] += time.perf_counter() - t0
            if pending is not None:  # collect the previous batch while the new one runs
                p_msgs, p_texts, p_slot, p_t = pending
                t0 = time.perf_counter()
                score, idx = index.search_host_wait(p_slot)
                self.stats["search_seconds"] += time.perf_counter() - t0
                self._emit_results(p_texts, score, idx)
                self.producer.flush()
                c.commit_offsets(p_msgs)
                self._note_latency(p_t, len(p_texts))
                pending = None
            if batch is None:
                break
            msgs, texts, vecs = batch
            if len(texts) and pipelined:
                pending = (msgs, texts, slot, time.perf_counter())
                slot ^= 1
            else:
                if len(texts):
                    t0 = time.perf_counter()
                    score, idx = index.search_host(vecs, self.k)
                    self.stats["search_seconds"] += time.perf_counter() - t0
                    self._emit_results(texts, score, idx)
                    self._note_latency(t0, len(texts))
                self.producer.flush()  # also carries any quarantined records of this batch
                c.commit_offsets(msgs)
        return total

    def stage_response(self) -> int:
        c, msgs, recs = self._drain("search_results")
        for m, r in recs:
            out = dict(r)
            out["response"] = self.generator(rag_prompt(r), r)
            self.producer.produce("search_results_response", value=self.codec.encode("search_results_response", out))
            self.stats["responses"] += 1
        if msgs:
            self.producer.flush()
            c.commit()
        return len(msgs)

    # ------------------------------------------------------------------ loop
    def run_once(self) -> int:
        """One pass over all stages in topological order; returns the number of records moved.  The ingest stages
        are drained completely first, so a query is searched against every document that was already on the
        log when the pass started (Flink gives no such ordering across topics; this is strictly stronger)."""
        moved = 0
        while True:
            n = self.stage_documents() + self.stage_sink()
            moved += n
            if n == 0:
                break
        moved += self.stage_queries() + self.stage_search() + self.stage_response()
        for st in self.extra_stages:
            moved += st.run_once()
        return moved

    def run_until_idle(self, max_passes: int = 1000) -> int:
        total = 0
        for _ in range(max_passes):
            n = self.run_once()
            total += n
            if n == 0:
                break
        return total

    def snapshot(self, directory: str) -> int:
        """Checkpoint the table together with the `documents_embed` offsets its content reaches (everything the sink has
        consumed is in the table by the time a stage returns).  Written atomically; see VectorTable.save."""
        pos = self.consumers["documents_embed"].positions("documents_embed")
        n = self.table.save(directory, {f"documents_embed-{p}": o for p, o in pos.items()})
        self.stats["snapshots"] += 1
        self._sink_dirty = False
        return n

    def run_forever(self, idle_sleep: float = 0.05, stop=lambda: False, snapshot_dir: str | None = None,
                    snapshot_every_s: float = 30.0) -> None:
        last = time.time()
        while not stop():
            if self.run_once() == 0:
                time.sleep(idle_sleep)
            if snapshot_dir and self._sink_dirty and time.time() - last >= snapshot_every_s:
                self.snapshot(snapshot_dir)
                last = time.time()
