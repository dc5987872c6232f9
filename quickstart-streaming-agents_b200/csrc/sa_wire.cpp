// Host-side batch codecs of libsa_b200.so (include/sa_wire.h): the records either side of the search, decoded /
// encoded a batch at a time with no per-record interpreter work.  Formats: SURVEY.md appendix C (Confluent framing
// scripts/publish_lab3_data.py:96-122; Avro binary rules; Flink's nullable-union schemas, main.tf:141,292).
#include "../../include/sa_api.h"
#include "../../include/sa_wire.h"

#include <algorithm>
#include <cmath>
#include <cstdlib>
#include <cstring>
#include <thread>
#include <vector>

extern "C" int sa_internal_fail(int rc, const char* fmt, ...);  // sa_api.cu: sets sa_last_error()

namespace {

constexpr uint32_t kNullLen = 0xFFFFFFFFu;

// `dim` items of an Avro array of ["null","float"]: true iff every item is the float branch (byte 2) and finite; the
// floats land in dst.  No early exit, so the loop unrolls and pipelines (a batch of 1024 x 1536-d embeddings is 1.6 M
// items: this loop is the decode).  The caller has checked that 5 * dim bytes are readable and zero-fills dst on failure.
inline bool copy_float_items(const uint8_t* p, int dim, float* dst) {
  uint32_t bad = 0;
  for (int j = 0; j < dim; ++j) {
    uint32_t bits;
    memcpy(&bits, p + 5 * static_cast<size_t>(j) + 1, 4);
    bad |= static_cast<uint32_t>(p[5 * static_cast<size_t>(j)] ^ 2u);
    bad |= static_cast<uint32_t>((bits & 0x7F800000u) == 0x7F800000u);   // inf or NaN
    memcpy(dst + j, &bits, 4);
  }
  return bad == 0;
}

// Strict UTF-8 (what Python's bytes.decode("utf-8") accepts: no overlong forms, no surrogates, nothing above U+10FFFF).
// A string the generic codec would refuse to decode must not pass here either -- the record is then handed over and
// quarantined there, instead of travelling on as bytes nobody can decode.
inline bool valid_utf8(const uint8_t* s, size_t n) {
  size_t i = 0;
  while (i < n) {
    if (i + 8 <= n) {  // eight ASCII bytes at a time
      uint64_t w;
      memcpy(&w, s + i, 8);
      if (!(w & 0x8080808080808080ull)) {
        i += 8;
        continue;
      }
    }
    const uint8_t c = s[i];
    if (c < 0x80) {
      ++i;
    } else if (c < 0xC2) {
      return false;  // a continuation byte, or the lead of an overlong two-byte form
    } else if (c < 0xE0) {
      if (i + 1 >= n || (s[i + 1] & 0xC0) != 0x80) return false;
      i += 2;
    } else if (c < 0xF0) {
      if (i + 2 >= n || (s[i + 1] & 0xC0) != 0x80 || (s[i + 2] & 0xC0) != 0x80) return false;
      if (c == 0xE0 && s[i + 1] < 0xA0) return false;   // overlong
      if (c == 0xED && s[i + 1] >= 0xA0) return false;  // UTF-16 surrogates
      i += 3;
    } else if (c < 0xF5) {
      if (i + 3 >= n || (s[i + 1] & 0xC0) != 0x80 || (s[i + 2] & 0xC0) != 0x80 || (s[i + 3] & 0xC0) != 0x80) return false;
      if (c == 0xF0 && s[i + 1] < 0x90) return false;   // overlong
      if (c == 0xF4 && s[i + 1] >= 0x90) return false;  // above U+10FFFF
      i += 4;
    } else {
      return false;
    }
  }
  return true;
}

// Records of a batch are independent: decode them on a few threads (SA_WIRE_THREADS, default 4; small batches stay on
// the caller's thread).  Plain std::thread -- OpenMP would be pinned to one thread by torchrun's OMP_NUM_THREADS=1.
int wire_threads() {
  static const int n = [] {
    const char* e = getenv("SA_WIRE_THREADS");
    int v = e ? atoi(e) : 4;
    const unsigned hw = std::thread::hardware_concurrency();
    if (hw > 0) v = std::min<int>(v, static_cast<int>(hw));
    return std::max(1, std::min(v, 16));
  }();
  return n;
}
template <typename F>
void for_each_record(int n, F&& body) {   // body(first, last)
  const int t = (n >= 256) ? std::min(wire_threads(), n / 128) : 1;
  if (t <= 1) {
    body(0, n);
    return;
  }
  std::vector<std::thread> th;
  th.reserve(t - 1);
  const int per = (n + t - 1) / t;
  for (int i = 1; i < t; ++i) {
    const int lo = std::min(n, i * per), hi = std::min(n, (i + 1) * per);
    if (lo < hi) th.emplace_back([&body, lo, hi] { body(lo, hi); });
  }
  body(0, std::min(n, per));
  for (auto& x : th) x.join();
}

inline uint32_t rd_u32(const uint8_t* p) {
  uint32_t v;
  memcpy(&v, p, 4);
  return v;
}
inline void wr_u32(uint8_t* p, uint32_t v) { memcpy(p, &v, 4); }
inline void wr_i64(uint8_t* p, int64_t v) { memcpy(p, &v, 8); }

// Avro long: zig-zag, base-128 little-endian groups.  Returns false on truncation / overlong encoding.
inline bool read_long(const uint8_t* p, const uint8_t* end, int64_t* out, const uint8_t** next) {
  uint64_t u = 0;
  int shift = 0;
  while (p < end && shift <= 63) {
    const uint8_t b = *p++;
    u |= static_cast<uint64_t>(b & 0x7F) << shift;
    if (!(b & 0x80)) {
      *out = static_cast<int64_t>(u >> 1) ^ -static_cast<int64_t>(u & 1);
      *next = p;
      return true;
    }
    shift += 7;
  }
  return false;
}
inline int long_size(int64_t v) {
  uint64_t u = (static_cast<uint64_t>(v) << 1) ^ static_cast<uint64_t>(v >> 63);
  int n = 1;
  while (u > 0x7F) {
    u >>= 7;
    ++n;
  }
  return n;
}
inline uint8_t* write_long(uint8_t* p, int64_t v) {
  uint64_t u = (static_cast<uint64_t>(v) << 1) ^ static_cast<uint64_t>(v >> 63);
  while (u > 0x7F) {
    *p++ = static_cast<uint8_t>((u & 0x7F) | 0x80);
    u >>= 7;
  }
  *p++ = static_cast<uint8_t>(u);
  return p;
}
inline uint8_t* write_header(uint8_t* p, uint32_t schema_id) {
  p[0] = 0;
  p[1] = static_cast<uint8_t>(schema_id >> 24);
  p[2] = static_cast<uint8_t>(schema_id >> 16);
  p[3] = static_cast<uint8_t>(schema_id >> 8);
  p[4] = static_cast<uint8_t>(schema_id);
  return p + 5;
}

}  // namespace

extern "C" {

int sa_wire_split_log(const uint8_t* buf, uint64_t buf_len, int n, uint64_t* value_off, uint32_t* value_len,
                      uint64_t* key_off, uint32_t* key_len, int64_t* timestamp_ms) {
  if (!buf || !value_off || !value_len || n < 0) return sa_internal_fail(SA_ERR_ARG, "sa_wire_split_log: null argument");
  uint64_t pos = 0;
  for (int i = 0; i < n; ++i) {
    if (pos + 4 > buf_len) return sa_internal_fail(SA_ERR_ARG, "log slice truncated in record %d", i);
    const uint32_t kl = rd_u32(buf + pos);
    pos += 4;
    if (key_off) key_off[i] = pos;
    if (key_len) key_len[i] = kl;
    if (kl != kNullLen) pos += kl;
    if (pos + 4 > buf_len) return sa_internal_fail(SA_ERR_ARG, "log slice truncated in record %d", i);
    const uint32_t vl = rd_u32(buf + pos);
    pos += 4;
    value_off[i] = pos;
    value_len[i] = vl;
    if (vl != kNullLen) pos += vl;
    if (pos + 8 > buf_len) return sa_internal_fail(SA_ERR_ARG, "log slice truncated in record %d", i);
    if (timestamp_ms) memcpy(&timestamp_ms[i], buf + pos, 8);
    pos += 8;
  }
  return SA_OK;
}

int sa_wire_decode_queries_embed(const uint8_t* buf, const uint64_t* value_off, const uint32_t* value_len, int n, int dim,
                                 uint32_t schema_id, float* out_vec, uint64_t* text_off, uint32_t* text_len,
                                 uint8_t* status, int* n_ok) {
  if (!buf || !value_off || !value_len || !out_vec || !text_off || !text_len || !status || n < 0 || dim <= 0)
    return sa_internal_fail(SA_ERR_ARG, "sa_wire_decode_queries_embed: bad argument");
  for_each_record(n, [&](int first, int last) {
  for (int i = first; i < last; ++i) {
    float* dst = out_vec + static_cast<size_t>(i) * dim;
    status[i] = 1;
    text_off[i] = 0;
    text_len[i] = 0;
    bool good = false;
    do {
      const uint32_t vl = value_len[i];
      if (vl == kNullLen || vl < 5) break;
      const uint8_t* p = buf + value_off[i];
      const uint8_t* end = p + vl;
      if (p[0] != 0) break;
      const uint32_t sid = (static_cast<uint32_t>(p[1]) << 24) | (static_cast<uint32_t>(p[2]) << 16) |
                           (static_cast<uint32_t>(p[3]) << 8) | p[4];
      if (sid != schema_id) break;
      p += 5;
      if (p >= end || *p++ != 2) break;  // query: ["null","string"], branch 1
      int64_t tl;
      if (!read_long(p, end, &tl, &p) || tl < 0 || tl > end - p) break;
      const uint8_t* text = p;
      if (!valid_utf8(text, static_cast<size_t>(tl))) break;
      p += tl;
      if (p >= end || *p++ != 2) break;  // embedding: ["null", array], branch 1
      int64_t cnt;
      if (!read_long(p, end, &cnt, &p) || cnt != dim) break;  // one block of exactly dim items
      if (end - p != static_cast<int64_t>(dim) * 5 + 1) break;
      if (!copy_float_items(p, dim, dst)) break;  // a null item or a non-finite value
      p += static_cast<size_t>(dim) * 5;
      if (*p != 0) break;  // end-of-array marker
      text_off[i] = static_cast<uint64_t>(text - buf);
      text_len[i] = static_cast<uint32_t>(tl);
      good = true;
    } while (false);
    if (good)
      status[i] = 0;
    else
      memset(dst, 0, sizeof(float) * dim);
  }
  });
  if (n_ok) {
    int ok = 0;
    for (int i = 0; i < n; ++i) ok += status[i] == 0;
    *n_ok = ok;
  }
  return SA_OK;
}

namespace {
// Skip one Avro value of the shapes the metadata columns have; false = malformed / truncated.
inline bool skip_nullable_string(const uint8_t*& p, const uint8_t* end) {
  int64_t br;
  if (!read_long(p, end, &br, &p)) return false;
  if (br == 0) return true;
  if (br != 1) return false;
  int64_t n;
  if (!read_long(p, end, &n, &p) || n < 0 || n > end - p) return false;
  if (!valid_utf8(p, static_cast<size_t>(n))) return false;
  p += n;
  return true;
}
inline bool skip_nullable_string_array(const uint8_t*& p, const uint8_t* end) {
  int64_t br;
  if (!read_long(p, end, &br, &p)) return false;
  if (br == 0) return true;
  if (br != 1) return false;
  for (;;) {
    int64_t cnt;
    if (!read_long(p, end, &cnt, &p)) return false;
    if (cnt == 0) return true;
    if (cnt < 0) {
      int64_t bytes;
      if (!read_long(p, end, &bytes, &p)) return false;
      cnt = -cnt;
    }
    for (int64_t i = 0; i < cnt; ++i)
      if (!skip_nullable_string(p, end)) return false;
  }
}
inline bool skip_nullable_int(const uint8_t*& p, const uint8_t* end) {
  int64_t br, v;
  if (!read_long(p, end, &br, &p)) return false;
  if (br == 0) return true;
  return br == 1 && read_long(p, end, &v, &p);
}
}  // namespace

int sa_wire_decode_documents_embed(const uint8_t* buf, const uint64_t* value_off, const uint32_t* value_len, int n, int dim,
                                   uint32_t schema_id, float* out_vec, uint64_t* id_off, uint32_t* id_len,
                                   uint64_t* chunk_off, uint32_t* chunk_len, uint64_t* meta_off, uint32_t* meta_len,
                                   uint8_t* status, int* n_ok) {
  if (!buf || !value_off || !value_len || !out_vec || !id_off || !id_len || !chunk_off || !chunk_len || !meta_off ||
      !meta_len || !status || n < 0 || dim <= 0)
    return sa_internal_fail(SA_ERR_ARG, "sa_wire_decode_documents_embed: bad argument");
  for_each_record(n, [&](int first, int last) {
  for (int i = first; i < last; ++i) {
    float* dst = out_vec + static_cast<size_t>(i) * dim;
    status[i] = 1;
    id_off[i] = chunk_off[i] = meta_off[i] = 0;
    id_len[i] = chunk_len[i] = kNullLen;
    meta_len[i] = 0;
    bool good = false;
    do {
      const uint32_t vl = value_len[i];
      if (vl == kNullLen || vl < 5) break;
      const uint8_t* p = buf + value_off[i];
      const uint8_t* end = p + vl;
      if (p[0] != 0) break;
      const uint32_t sid = (static_cast<uint32_t>(p[1]) << 24) | (static_cast<uint32_t>(p[2]) << 16) |
                           (static_cast<uint32_t>(p[3]) << 8) | p[4];
      if (sid != schema_id) break;
      p += 5;
      // document_id, chunk: ["null","string"] (either may be null)
      uint64_t so[2];
      uint32_t sl[2];
      bool strings_ok = true;
      for (int f = 0; f < 2; ++f) {
        int64_t br;
        if (!read_long(p, end, &br, &p) || (br != 0 && br != 1)) {
          strings_ok = false;
          break;
        }
        so[f] = 0;
        sl[f] = kNullLen;
        if (br == 1) {
          int64_t tl;
          if (!read_long(p, end, &tl, &p) || tl < 0 || tl > end - p || !valid_utf8(p, static_cast<size_t>(tl))) {
            strings_ok = false;
            break;
          }
          so[f] = static_cast<uint64_t>(p - buf);
          sl[f] = static_cast<uint32_t>(tl);
          p += tl;
        }
      }
      if (!strings_ok) break;
      // embedding: one block of exactly dim non-null finite floats
      if (p >= end || *p++ != 2) break;
      int64_t cnt;
      if (!read_long(p, end, &cnt, &p) || cnt != dim) break;
      if (end - p < static_cast<int64_t>(dim) * 5 + 1) break;
      if (!copy_float_items(p, dim, dst)) break;
      p += static_cast<size_t>(dim) * 5;
      if (*p++ != 0) break;
      // metadata columns (terraform/lab4-pubsec-fraud-agents/main.tf:271-289): validated here, decoded lazily by the host
      const uint8_t* m0 = p;
      if (!skip_nullable_string(p, end) || !skip_nullable_string(p, end) || !skip_nullable_string(p, end) ||
          !skip_nullable_string_array(p, end) || !skip_nullable_string_array(p, end) || !skip_nullable_int(p, end))
        break;
      if (p != end) break;
      id_off[i] = so[0];
      id_len[i] = sl[0];
      chunk_off[i] = so[1];
      chunk_len[i] = sl[1];
      meta_off[i] = static_cast<uint64_t>(m0 - buf);
      meta_len[i] = static_cast<uint32_t>(end - m0);
      good = true;
    } while (false);
    if (good)
      status[i] = 0;
    else
      memset(dst, 0, sizeof(float) * dim);
  }
  });
  if (n_ok) {
    int ok = 0;
    for (int i = 0; i < n; ++i) ok += status[i] == 0;
    *n_ok = ok;
  }
  return SA_OK;
}

int sa_wire_encode_search_results(int n, int k, int n_out, uint32_t schema_id, const uint8_t* text_buf,
                                  const uint64_t* text_off, const uint32_t* text_len, const float* score,
                                  const int64_t* row, const uint8_t* doc_arena, const uint64_t* doc_off,
                                  const uint8_t* chunk_arena, const uint64_t* chunk_off, int64_t table_rows, int score_mode,
                                  int64_t ts_ms, uint8_t* out, uint64_t out_cap, uint64_t* out_rec_off, uint64_t* needed) {
  if (n < 0 || k <= 0 || n_out <= 0 || !text_off || !text_len || !score || !row || !doc_off || !chunk_off || !out_rec_off)
    return sa_internal_fail(SA_ERR_ARG, "sa_wire_encode_search_results: bad argument");
  // pass 1: sizes
  uint64_t total = 0;
  for (int i = 0; i < n; ++i) {
    uint64_t v = 5;
    v += text_len[i] == kNullLen ? 1 : 1 + long_size(text_len[i]) + text_len[i];
    for (int j = 0; j < n_out; ++j) {
      const int64_t r = j < k ? row[static_cast<size_t>(i) * k + j] : -1;
      if (r < 0) {
        v += 3;
      } else {
        if (r >= table_rows) return sa_internal_fail(SA_ERR_ARG, "result row %lld outside the table (%lld rows)", (long long)r, (long long)table_rows);
        v += (doc_off[r + 1] - doc_off[r]) + (chunk_off[r + 1] - chunk_off[r]) + 9;
      }
    }
    out_rec_off[i] = total;
    total += 4 + 4 + v + 8;
  }
  out_rec_off[n] = total;
  if (needed) *needed = total;
  if (total > out_cap || !out) return sa_internal_fail(SA_ERR_CAPACITY, "output buffer too small: need %llu bytes", (unsigned long long)total);
  // pass 2: bytes
  for (int i = 0; i < n; ++i) {
    uint8_t* p = out + out_rec_off[i];
    const uint32_t vlen = static_cast<uint32_t>(out_rec_off[i + 1] - out_rec_off[i] - 16);
    wr_u32(p, kNullLen);
    wr_u32(p + 4, vlen);
    p = write_header(p + 8, schema_id);
    if (text_len[i] == kNullLen) {
      *p++ = 0;
    } else {
      *p++ = 2;
      p = write_long(p, text_len[i]);
      memcpy(p, text_buf + text_off[i], text_len[i]);
      p += text_len[i];
    }
    for (int j = 0; j < n_out; ++j) {
      const int64_t r = j < k ? row[static_cast<size_t>(i) * k + j] : -1;
      if (r < 0) {
        *p++ = 0;
        *p++ = 0;
        *p++ = 0;
        continue;
      }
      uint64_t len = doc_off[r + 1] - doc_off[r];
      memcpy(p, doc_arena + doc_off[r], len);
      p += len;
      len = chunk_off[r + 1] - chunk_off[r];
      memcpy(p, chunk_arena + chunk_off[r], len);
      p += len;
      double s = static_cast<double>(score[static_cast<size_t>(i) * k + j]);
      if (score_mode == 1) s = 0.5 * (1.0 + s);
      else if (score_mode == 2) s = 1.0 / (1.0 + s);
      *p++ = 2;
      memcpy(p, &s, 8);
      p += 8;
    }
    wr_i64(p, ts_ms);
  }
  return SA_OK;
}

int sa_wire_encode_queries_embed(int n, int dim, uint32_t schema_id, const uint8_t* text_buf, const uint64_t* text_off,
                                 const uint32_t* text_len, const float* vec, int64_t ts_ms, uint8_t* out, uint64_t out_cap,
                                 uint64_t* out_rec_off, uint64_t* needed) {
  if (n < 0 || dim <= 0 || !text_off || !text_len || !vec || !out_rec_off)
    return sa_internal_fail(SA_ERR_ARG, "sa_wire_encode_queries_embed: bad argument");
  uint64_t total = 0;
  for (int i = 0; i < n; ++i) {
    out_rec_off[i] = total;
    const uint64_t v = 5 + 1 + long_size(text_len[i]) + text_len[i] + 1 + long_size(dim) + static_cast<uint64_t>(dim) * 5 + 1;
    total += 4 + 4 + v + 8;
  }
  out_rec_off[n] = total;
  if (needed) *needed = total;
  if (total > out_cap || !out) return sa_internal_fail(SA_ERR_CAPACITY, "output buffer too small: need %llu bytes", (unsigned long long)total);
  for (int i = 0; i < n; ++i) {
    uint8_t* p = out + out_rec_off[i];
    wr_u32(p, kNullLen);
    wr_u32(p + 4, static_cast<uint32_t>(out_rec_off[i + 1] - out_rec_off[i] - 16));
    p = write_header(p + 8, schema_id);
    *p++ = 2;
    p = write_long(p, text_len[i]);
    memcpy(p, text_buf + text_off[i], text_len[i]);
    p += text_len[i];
    *p++ = 2;
    p = write_long(p, dim);
    const float* v = vec + static_cast<size_t>(i) * dim;
    for (int j = 0; j < dim; ++j) {
      *p++ = 2;
      memcpy(p, v + j, 4);
      p += 4;
    }
    *p++ = 0;
    wr_i64(p, ts_ms);
  }
  return SA_OK;
}

}  // extern "C"
