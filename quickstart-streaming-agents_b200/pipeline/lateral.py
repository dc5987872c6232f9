"""The operator's other two call sites: ``VECTOR_SEARCH_AGG`` applied per row of an upstream stream.

Lab2 searches a topic of bare queries (pipeline/serve.py).  Lab3 and Lab4 join the operator LATERALly onto a stream that
carries its own columns, embed one of them, and project the hits next to the carried columns
(LAB3-Walkthrough.md:225-375, LAB4-Walkthrough.md:251-309):

    SELECT c.<carried columns>, vs.search_results[i].<table column> AS <prefix>_i, ...
    FROM <upstream with a text column> c,
         LATERAL TABLE(ML_PREDICT('llm_embedding_model', c.<text>)) e,
         LATERAL TABLE(VECTOR_SEARCH_AGG(<vector table>, DESCRIPTOR(embedding), e.embedding, 3)) vs

``LateralSearch`` is that statement as a consumer/producer stage over the same transports as the Lab2 loop: records of
``source_topic`` are decoded with the schema their id names, filtered (``where``), embedded (stub, or taken from
``vector_field`` when the upstream already carries a vector), searched in one batch through the engine's host path, and
written to ``sink_topic`` under a schema derived from the source's (carried columns keep their types; projected columns
get the vector table's column types; ``score`` is a double).  At-least-once, poison records to ``<source>.dlq``.

``lab3_anomalies_enriched`` and ``lab4_claims_with_policies`` are the two statements of the reference with their column
lists, query text and prompt restated; the LLM call (``ml_predict('llm_textgen_model', ...)``) is a stub, as in Lab2.
"""
from __future__ import annotations

import datetime as _dt
import logging
import struct

import numpy as np

from ..embed.stub import StubEmbedder
from ..operator import SearchHit, VectorTable, atlas_score, project_search_results
from ..wire import avro, schemas
from ..wire.registry import SchemaRegistry

log = logging.getLogger(__name__)

_NULL_STRING = ["null", "string"]


def _table_column_type(col: str):
    """Avro type of a vector-table column as it appears in a projection (nullable: a query may have fewer than n hits)."""
    if col == "score":
        return ["null", "double"]
    for f in schemas.DOCUMENTS_EMBED_VALUE["fields"]:
        if f["name"] == col and col != "embedding":
            return f["type"] if isinstance(f["type"], list) else ["null", f["type"]]
    raise ValueError(f"the vector table has no column {col!r} to project")


class LateralSearch:
    def __init__(self, log_dir: str, table: VectorTable, source_topic: str, sink_topic: str, *, columns: dict[str, str],
                 k: int = 3, n_out: int | None = None, vector_field: str | None = "embedding", text_field: str | None = None,
                 query_builder=None, query_field: str | None = None, carry=None, where=None, select=None,
                 response_field: str | None = None, prompt_builder=None, generator=None, embedder=None,
                 score_mode: str = "cosine", max_batch: int = 1024, group: str = "sa-lateral", transport=None,
                 client_conf: dict | None = None):
        """``columns``: vector-table column -> output prefix (``{"chunk": "policy_chunk"}`` yields policy_chunk_1..n), in
        the order they are to appear per hit.  The query vector of a row is ``row[vector_field]`` when present and not
        null, else the embedding of ``query_builder(row)`` / ``row[text_field]``.  ``carry``: upstream columns copied to
        the output (default: all but the vector).  ``query_field``: also emit the query text under this name.
        ``response_field`` + ``prompt_builder`` + ``generator``: append the text generator's answer (ml_predict stub).
        ``select``: final column list (the outer SELECT), default everything in the order built.  ``k`` is at most the
        index's max_k (up to 64); ``n_out`` (default k) hits per row are projected."""
        if score_mode not in ("cosine", "atlas"):
            raise ValueError("score_mode must be 'cosine' or 'atlas'")
        if text_field is None and query_builder is None and vector_field is None:
            raise ValueError("nothing to search with: give vector_field, text_field or query_builder")
        if response_field and not (prompt_builder and generator):
            raise ValueError("response_field needs prompt_builder and generator")
        for c in columns:
            _table_column_type(c)
        self.table, self.k, self.n_out = table, int(k), int(n_out or k)
        if self.n_out > self.k:
            raise ValueError("n_out cannot exceed k")
        self.source_topic, self.sink_topic = source_topic, sink_topic
        self.columns, self.carry, self.where, self.select = dict(columns), carry, where, select
        self.vector_field, self.text_field, self.query_builder, self.query_field = vector_field, text_field, query_builder, query_field
        self.response_field, self.prompt_builder, self.generator = response_field, prompt_builder, generator
        self.embedder = embedder or StubEmbedder(table.index.dim)
        self.score_mode, self.max_batch = score_mode, max_batch
        self.registry = SchemaRegistry(log_dir)
        tp_mod = transport
        if tp_mod is None:
            from ..transport import filelog as tp_mod
        base = dict(client_conf or {})
        base["log.dir"] = log_dir
        self.producer = tp_mod.Producer(base)
        self.consumer = tp_mod.Consumer(dict(base, **{"group.id": group, "auto.offset.reset": "earliest",
                                                      "enable.auto.commit": False}))
        self.consumer.subscribe([source_topic])
        self._dec: dict[int, avro.CompiledSchema] = {}
        self._enc: dict[int, tuple[bytes, avro.CompiledSchema, list[str], list[str]]] = {}
        self.stats = {"rows": 0, "searched": 0, "filtered": 0, "quarantined": 0}

    # ------------------------------------------------------------------ schemas
    def sink_schema(self, source_schema) -> tuple[dict, list[str]]:
        """The output record type for rows of ``source_schema``, and the carried column names."""
        src = {f["name"]: f for f in source_schema["fields"]}
        carried = list(self.carry) if self.carry is not None else [n for n in src if n != self.vector_field]
        missing = [c for c in carried if c not in src]
        if missing:
            raise avro.AvroError(f"{self.source_topic} has no column(s) {missing}")
        fields = [{"name": c, "type": src[c]["type"], **({"default": src[c]["default"]} if "default" in src[c] else {})}
                  for c in carried]
        if self.query_field:
            fields.append({"name": self.query_field, "type": _NULL_STRING, "default": None})
        for i in range(1, self.n_out + 1):
            for col, prefix in self.columns.items():
                fields.append({"name": f"{prefix}_{i}", "type": _table_column_type(col), "default": None})
        if self.response_field:
            fields.append({"name": self.response_field, "type": _NULL_STRING, "default": None})
        if self.select is not None:
            by_name = {f["name"]: f for f in fields}
            unknown = [c for c in self.select if c not in by_name]
            if unknown:
                raise ValueError(f"select names column(s) the statement does not produce: {unknown}")
            fields = [by_name[c] for c in self.select]
        return ({"type": "record", "name": f"{self.sink_topic}_value", "namespace": schemas.NAMESPACE, "fields": fields},
                carried)

    def _encoder_for(self, sid: int):
        e = self._enc.get(sid)
        if e is None:
            schema, carried = self.sink_schema(self.registry.get(sid))
            out_id = self.registry.register(f"{self.sink_topic}-value", schema)
            e = self._enc[sid] = (avro.frame(out_id, b""), avro.CompiledSchema(schema), carried,
                                  [f["name"] for f in schema["fields"]])
        return e

    def _decode(self, raw: bytes):
        if raw is None or len(raw) < 5:
            raise avro.AvroError(f"Avro payload too short ({0 if raw is None else len(raw)} bytes)")
        if raw[0] != avro.MAGIC:
            raise avro.AvroError(f"Invalid Avro magic byte: {raw[0]}")
        sid = struct.unpack_from(">I", raw, 1)[0]
        cs = self._dec.get(sid)
        if cs is None:
            cs = self._dec[sid] = avro.CompiledSchema(self.registry.get(sid))
        return sid, cs.decode(raw, 5)

    def _quarantine(self, m, why: str) -> None:
        self.stats["quarantined"] += 1
        log.warning("quarantined %s[%d]@%d: %s", self.source_topic, m.partition(), m.offset(), why)
        self.producer.produce(f"{self.source_topic}.dlq", key=why, value=m.value())

    # ------------------------------------------------------------------ the stage
    def run_once(self) -> int:
        msgs = self.consumer.consume(self.max_batch, 0.0)
        if not msgs:
            return 0
        dim = self.table.index.dim
        rows = []  # (message, source schema id, record, query text)
        vecs = []
        for m in msgs:
            try:
                sid, rec = self._decode(m.value())
                self._encoder_for(sid)
                if self.where is not None and not self.where(rec):
                    self.stats["filtered"] += 1
                    continue
                text = None
                if self.query_builder is not None:
                    text = self.query_builder(rec)
                elif self.text_field is not None:
                    text = rec.get(self.text_field)
                vec = rec.get(self.vector_field) if self.vector_field else None
                if vec is None:
                    if text is None:
                        raise avro.AvroError("row has neither a query vector nor a text to embed")
                    vec = self.embedder.embed(text)
                vec = np.asarray(vec, dtype=np.float32)
                if vec.shape != (dim,) or not np.isfinite(vec).all():
                    raise avro.AvroError(f"embedding must be {dim} finite floats")
            except Exception as e:  # poison record: quarantine, keep going
                self._quarantine(m, str(e))
                continue
            rows.append((m, sid, rec, text))
            vecs.append(vec)
        if rows:
            score, idx = self.table.index.search_host(np.ascontiguousarray(np.stack(vecs), dtype=np.float32), self.k)
            t = self.table
            for r, (m, sid, rec, text) in enumerate(rows):
                hits = []
                for s, i in zip(score[r].tolist(), idx[r].tolist()):
                    if i < 0:
                        break
                    s = atlas_score(s, t.similarity) if self.score_mode == "atlas" else s
                    hits.append(SearchHit(t.document_id[i], t.chunk[i], float(s), int(i), t.metadata[i]))
                header, cs, carried, names = self._enc[sid]
                out = {c: rec.get(c) for c in carried}
                if self.query_field:
                    out[self.query_field] = text
                out.update(project_search_results(hits, self.columns, self.n_out))
                if self.response_field:
                    out[self.response_field] = self.generator(self.prompt_builder(out), out)
                self.producer.produce(self.sink_topic, key=m.key(), value=cs.encode({n: out.get(n) for n in names}, prefix=header))
            self.stats["searched"] += len(rows)
        self.stats["rows"] += len(msgs)
        self.producer.flush()
        self.consumer.commit_offsets(msgs)
        return len(msgs)

    def run_until_idle(self, max_passes: int = 1000) -> int:
        total = 0
        for _ in range(max_passes):
            n = self.run_once()
            total += n
            if n == 0:
                break
        return total


# ---------------------------------------------------------------------------------------------------------------------
# Lab3: anomalies_per_zone -> anomalies_enriched (LAB3-Walkthrough.md:225-375)
# ---------------------------------------------------------------------------------------------------------------------
_DAY_PARTS = (  # CASE WHEN HOUR(window_time) ... (LAB3-Walkthrough.md:279-289)
    (0, 4, "late night hours (12:00 AM - 4:00 AM)"),
    (4, 7, "early morning setup period (4:00 AM - 7:00 AM)"),
    (7, 9, "morning rush hours (7:00 AM - 9:00 AM)"),
    (9, 12, "late morning period (9:00 AM - 12:00 PM)"),
    (12, 14, "lunch service peak (12:00 PM - 2:00 PM)"),
    (14, 17, "afternoon hours (2:00 PM - 5:00 PM)"),
    (17, 20, "evening dinner period (5:00 PM - 8:00 PM)"),
    (20, 23, "nightlife hours (8:00 PM - 11:00 PM)"),
)


def _as_datetime(ts, tz) -> _dt.datetime:
    if isinstance(ts, _dt.datetime):
        return ts.astimezone(tz) if ts.tzinfo else ts.replace(tzinfo=_dt.timezone.utc).astimezone(tz)
    return _dt.datetime.fromtimestamp(int(ts) / 1000.0, tz=_dt.timezone.utc).astimezone(tz)   # timestamp-millis


def _h_mm_a(t: _dt.datetime) -> str:            # DATE_FORMAT(ts, 'h:mm a')
    return f"{(t.hour % 12) or 12}:{t.minute:02d} {'AM' if t.hour < 12 else 'PM'}"


def _sql_string(v) -> str:                      # CAST(x AS STRING) for the numeric types that occur here
    if isinstance(v, bool):
        return "TRUE" if v else "FALSE"
    if isinstance(v, int):
        return str(v)
    return repr(float(v))


def surge_query(row: dict, tz=_dt.timezone.utc) -> str:
    """The query text Lab3 embeds for a surge window (the CONCAT of LAB3-Walkthrough.md:270-311).  ``window_time`` is a
    timestamp-millis (rendered in ``tz``; Flink renders TIMESTAMP_LTZ in the session time zone)."""
    t = _as_datetime(row["window_time"], tz)
    part = next((name for lo, hi, name in _DAY_PARTS if lo <= t.hour < hi), "late night period (11:00 PM - 12:00 AM)")
    exp, act = row["expected_requests"], row["request_count"]
    pct = round(((act - exp) / exp) * 100, 1)
    hour = _dt.timedelta(hours=1)
    return ("Transportation demand surge in " + row["pickup_zone"] + " at " + _h_mm_a(t) + " (" + f"{t.hour:02d}:{t.minute:02d}" +
            ") during " + part + ". Looking for HIGH demand events occurring between " + _h_mm_a(t - hour) + " and " +
            _h_mm_a(t + hour) + ". Expected: " + _sql_string(exp) + ", Actual: " + _sql_string(act) + " (+" + _sql_string(pct) +
            "%). What HIGH impact events, festivals, or gatherings are active in " + row["pickup_zone"] + " during this time?")


def surge_prompt(rec: dict) -> str:
    """The prompt of LAB3-Walkthrough.md:355-371 over the searched row."""
    def s(v):
        return "" if v is None else (_sql_string(v) if isinstance(v, float) else str(v))
    head = ("Analyze the retrieved event documents and identify the most likely cause of this transportation demand surge. "
            "If a retrieved document describes an event with time ranges that overlap the surge time, cite it by name, "
            "attendance, and time. If no document is a strong match, describe the surge itself: the zone, the time of day, "
            "and the magnitude. Always provide a concise 1-2 sentence answer that gives the dispatch agent enough context to "
            "act. Do not say \"no events found\" — always produce a reason.\n\n")
    body = "USER QUERY: " + s(rec.get("query")) + "\n\nRETRIEVED DOCUMENTS:\n"
    for i in (1, 2, 3):
        body += (f"Document {i} (Score: " + s(rec.get(f"top_score_{i}")) + "):\nSource: " + s(rec.get(f"top_document_{i}")) + "\n" +
                 s(rec.get(f"top_chunk_{i}")) + "\n\n")
    return head + body + "Provide only the reason, no additional text."


def stub_reason(prompt: str, rec: dict) -> str:
    """Stand-in for ml_predict('llm_textgen_model', prompt): a deterministic one-sentence reason citing the best hit."""
    if rec.get("top_document_1") is None:
        return f"Demand surge in {rec.get('pickup_zone')}: {rec.get('request_count')} requests against {rec.get('expected_requests')} expected."
    chunk = (rec.get("top_chunk_1") or "").strip().replace("\n", " ")
    return f"Likely cause per {rec['top_document_1']}: {chunk[:200]}"


ANOMALIES_PER_ZONE_VALUE = {   # the columns the Lab3 statement reads from anomalies_per_zone (LAB3-Walkthrough.md:147-222)
    "type": "record", "name": "anomalies_per_zone_value", "namespace": schemas.NAMESPACE,
    "fields": [
        {"name": "pickup_zone", "type": "string"},
        {"name": "window_time", "type": {"type": "long", "logicalType": "timestamp-millis"}},
        {"name": "request_count", "type": "long"},
        {"name": "expected_requests", "type": ["null", "double"], "default": None},
        {"name": "is_surge", "type": ["null", "boolean"], "default": None},
    ],
}


def lab3_anomalies_enriched(log_dir: str, table: VectorTable, generator=stub_reason, **kw) -> LateralSearch:
    """``CREATE TABLE anomalies_enriched AS SELECT pickup_zone, window_time, request_count, expected_requests,
    anomaly_reason, top_chunk_1..3 ...`` (LAB3-Walkthrough.md:225-375) over documents_vectordb_lab3."""
    return LateralSearch(
        log_dir, table, "anomalies_per_zone", "anomalies_enriched",
        where=lambda r: r.get("is_surge") is True, query_builder=surge_query, query_field="query", vector_field=None,
        carry=("pickup_zone", "window_time", "request_count", "expected_requests", "is_surge"),
        columns={"document_id": "top_document", "chunk": "top_chunk", "score": "top_score"}, k=3,
        response_field="anomaly_reason", prompt_builder=surge_prompt, generator=generator,
        select=("pickup_zone", "window_time", "request_count", "expected_requests", "anomaly_reason",
                "top_chunk_1", "top_chunk_2", "top_chunk_3"), **kw)


# ---------------------------------------------------------------------------------------------------------------------
# Lab4: claims_to_investigate -> claims_to_investigate_with_policies (LAB4-Walkthrough.md:251-309)
# ---------------------------------------------------------------------------------------------------------------------
def _s(name, nullable=True):
    return {"name": name, "type": _NULL_STRING, "default": None} if nullable else {"name": name, "type": "string"}


_TS = {"type": "long", "logicalType": "timestamp-millis"}

CLAIMS_TO_INVESTIGATE_VALUE = {   # claims columns typed as the datagen publishes them (scripts/lab4_datagen.py:100-123)
    "type": "record", "name": "claims_to_investigate_value", "namespace": schemas.NAMESPACE,   # + the join's three columns
    "fields": [
        _s("claim_id", False), _s("applicant_name"), _s("city", False), _s("claim_narrative"), _s("claim_amount", False),
        _s("damage_assessed"), _s("has_insurance"), _s("insurance_amount"), _s("is_primary_residence"),
        _s("assessment_date"), _s("disaster_date"), _s("assessment_source"), _s("shared_account"), _s("shared_phone"),
        _s("previous_claims_count"), _s("last_claim_date"), {"name": "claim_timestamp", "type": _TS},
        {"name": "anomaly_window_time", "type": ["null", _TS], "default": None},
        {"name": "anomaly_total_amount", "type": ["null", "double"], "default": None},
        {"name": "is_anomaly", "type": ["null", "boolean"], "default": None},
    ],
}

LAB4_POLICY_COLUMNS = {   # vs.search_results[i].<column> AS <prefix>_i (LAB4-Walkthrough.md:280-300)
    "chunk": "policy_chunk", "score": "policy_score", "pages": "policy_pages", "section_reference": "policy_section",
    "title": "policy_title", "fraud_categories": "policy_fraud_cats", "policy_keywords": "policy_keywords",
}


def lab4_claims_with_policies(log_dir: str, table: VectorTable, **kw) -> LateralSearch:
    """``CREATE TABLE claims_to_investigate_with_policies AS WITH embedded AS (...ML_PREDICT(..., c.claim_narrative))
    SELECT c.*, vs.search_results[i].chunk AS policy_chunk_i, ... FROM embedded c, LATERAL TABLE(VECTOR_SEARCH_AGG(
    fema_policies_vectordb, DESCRIPTOR(embedding), c.narrative_embedding, 3)) vs`` (LAB4-Walkthrough.md:251-309): the
    narrative is embedded unless the row already carries ``narrative_embedding``."""
    carry = ("claim_id", "applicant_name", "city", "claim_amount", "damage_assessed", "has_insurance", "insurance_amount",
             "is_primary_residence", "claim_narrative", "assessment_date", "disaster_date", "assessment_source",
             "shared_account", "shared_phone", "previous_claims_count", "last_claim_date", "claim_timestamp",
             "anomaly_window_time", "anomaly_total_amount", "is_anomaly")               # LAB4-Walkthrough.md:259-279
    return LateralSearch(log_dir, table, "claims_to_investigate", "claims_to_investigate_with_policies",
                         vector_field="narrative_embedding", text_field="claim_narrative", carry=carry,
                         columns=LAB4_POLICY_COLUMNS, k=3, **kw)
