/* sa_wire.h -- host-side batch codecs of libsa_b200.so for the two record types either side of the search
 * (SURVEY.md section 8f-1): Confluent-framed Avro `queries_embed` in, `search_results` out, and the record framing of the
 * file-log transport.  Plain C ABI, no CUDA involved; the buffers may be page-locked (sa_host_alloc) so that the decoded
 * embeddings are DMA'd to the GPU without another copy.
 *
 * Formats (all fixed by the reference, SURVEY.md appendix C):
 *   Confluent wire format  byte 0 = 0x00, bytes 1-4 = big-endian schema id, then the Avro binary body
 *                          (scripts/publish_lab3_data.py:96-122, testing/helpers/kafka_helper.py:74-75);
 *   queries_embed_value    {query: ["null","string"], embedding: ["null", {array, items ["null","float"]}]}
 *                          (Flink's nullable-union convention, terraform/lab2-vector-search/main.tf:141);
 *   search_results_value   {query, document_id_1..n, chunk_1..n: ["null","string"]; score_1..n: ["null","double"]}
 *                          (the projection of main.tf:292);
 *   file-log record        u32 key_len (0xFFFFFFFF = null) | key | u32 value_len | value | i64 timestamp_ms, little-endian
 *                          (quickstart-streaming-agents_b200/transport/filelog.py).
 * Every function returns 0 or a negative sa_status (sa_api.h); sa_last_error() has the detail.
 * The two batch decoders spread the records of a large batch over a few threads (environment SA_WIRE_THREADS, default 4,
 * 1 = the caller's thread only); the threads live only for the duration of the call.
 */
#ifndef SA_WIRE_H_
#define SA_WIRE_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* Split a contiguous slice of a topic-partition log into its records.  buf holds n records back to back starting at
 * the first one.  Outputs per record: byte offset (within buf) and length of the value; key offset/length (length
 * 0xFFFFFFFF = null key); timestamp.  Fails with SA_ERR_ARG if the slice is truncated or malformed. */
int sa_wire_split_log(const uint8_t* buf, uint64_t buf_len, int n, uint64_t* value_off, uint32_t* value_len,
                      uint64_t* key_off, uint32_t* key_len, int64_t* timestamp_ms);

/* Batch decode of queries_embed values.  For record i (value bytes buf[value_off[i] .. +value_len[i])):
 *   status[i] = 0  decoded: out_vec[i*dim .. +dim) holds the embedding, text_off/text_len[i] the UTF-8 query inside buf
 *               1  anything else -- an unusual but legal shape (null query / null embedding / multi-block array / other
 *                  schema id) or a bad record (bad magic, truncated, null item, wrong length, non-finite value): hand it
 *                  to the generic codec, which decodes it or names the reason it is quarantined for
 * Rows of out_vec belonging to records with status != 0 are zero-filled.  Returns the number of status-0 records
 * through *n_ok. */
int sa_wire_decode_queries_embed(const uint8_t* buf, const uint64_t* value_off, const uint32_t* value_len, int n, int dim,
                                 uint32_t schema_id, float* out_vec, uint64_t* text_off, uint32_t* text_len,
                                 uint8_t* status, int* n_ok);

/* Batch decode of documents_embed values (the ingest side: `documents -> documents_embed -> vector table`,
 * LAB2-Walkthrough.md:41-51; schema = document_id, chunk, embedding + Lab4's six metadata columns,
 * terraform/lab4-pubsec-fraud-agents/main.tf:271-289).  status as above (0 decoded / 1 hand to the generic codec).
 * For status-0 records: out_vec row = embedding; id_* / chunk_* = the UTF-8 text inside buf (len 0xFFFFFFFF = null);
 * meta_* = the bytes of the six metadata fields (validated, decoded lazily by the caller). */
int sa_wire_decode_documents_embed(const uint8_t* buf, const uint64_t* value_off, const uint32_t* value_len, int n, int dim,
                                   uint32_t schema_id, float* out_vec, uint64_t* id_off, uint32_t* id_len,
                                   uint64_t* chunk_off, uint32_t* chunk_len, uint64_t* meta_off, uint32_t* meta_len,
                                   uint8_t* status, int* n_ok);

/* Batch encode of search_results records, already framed for the file log (null key, timestamp ts_ms), ready to be
 * appended with one write.  Record i: query text = text_buf[text_off[i] .. +text_len[i]) (text_len 0xFFFFFFFF = null),
 * results j = 0 .. n_out-1 from score[i*k + j] / row[i*k + j] (row < 0 = no hit -> three nulls).  The non-vector columns
 * of the table come pre-serialised as Avro ["null","string"] values in two arenas: column value of table row r is
 * doc_arena[doc_off[r] .. doc_off[r+1]) and chunk_arena[chunk_off[r] .. chunk_off[r+1]).  score_mode 0 = the raw score,
 * 1 = Atlas's (1 + s) / 2 (cosine, dotProduct), 2 = Atlas's 1 / (1 + d) (euclidean distance d).  out_rec_off[i] receives the offset of record i inside out (out_rec_off[n] = total bytes).
 * Fails with SA_ERR_CAPACITY (and reports the needed size in *needed) when out_cap is too small. */
int sa_wire_encode_search_results(int n, int k, int n_out, uint32_t schema_id, const uint8_t* text_buf,
                                  const uint64_t* text_off, const uint32_t* text_len, const float* score,
                                  const int64_t* row, const uint8_t* doc_arena, const uint64_t* doc_off,
                                  const uint8_t* chunk_arena, const uint64_t* chunk_off, int64_t table_rows, int score_mode,
                                  int64_t ts_ms, uint8_t* out, uint64_t out_cap, uint64_t* out_rec_off, uint64_t* needed);

/* Batch encode of queries_embed records (the producer side: bench / load generators), framed for the file log.
 * Record i: query text_buf[text_off[i] .. +text_len[i]), embedding vec[i*dim .. +dim). */
int sa_wire_encode_queries_embed(int n, int dim, uint32_t schema_id, const uint8_t* text_buf, const uint64_t* text_off,
                                 const uint32_t* text_len, const float* vec, int64_t ts_ms, uint8_t* out, uint64_t out_cap,
                                 uint64_t* out_rec_off, uint64_t* needed);

#ifdef __cplusplus
}
#endif
#endif /* SA_WIRE_H_ */
