// Kernels either side of the scan: ingest (fp32 -> bf16 or int8 + row terms), candidate merge + exact
// rescoring, and the cross-shard merge that follows the all-gather.  All are HBM/latency-bound
// integer/byte work on CUDA cores: coalesced 16-byte accesses, one warp per row / one block per query.
#pragma once
#include <cstdint>
#include <cmath>
#include <cstring>

namespace sa {

// Bit casts usable on both sides of the compiler: the device path is the intrinsic, the host path (used only by the
// CPU unit tests through sa_debug_*) is a memcpy.
__host__ __device__ __forceinline__ unsigned f32_bits(float f) {
#ifdef __CUDA_ARCH__
  return __float_as_uint(f);
#else
  unsigned u;
  memcpy(&u, &f, sizeof u);
  return u;
#endif
}
__host__ __device__ __forceinline__ float bits_f32(unsigned u) {
#ifdef __CUDA_ARCH__
  return __uint_as_float(u);
#else
  float f;
  memcpy(&f, &u, sizeof f);
  return f;
#endif
}

// Order-preserving float <-> unsigned key (larger float <=> larger key; key 0 is below every float).  The scan's shared
// thresholds hold these keys, and the merge kernel's 64-bit keys (make_key) carry one in their high word.
__host__ __device__ __forceinline__ unsigned float_to_key(float f) {
  const unsigned u = f32_bits(f);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__host__ __device__ __forceinline__ float key_to_float(unsigned k) {
  return bits_f32((k & 0x80000000u) ? (k & 0x7fffffffu) : ~k);
}

__host__ __device__ __forceinline__ float bf16_bits_to_f32(uint32_t b) { return bits_f32(b << 16); }
// Round-to-nearest-even fp32 -> bf16 bit pattern (NaN kept quiet); same rule as the oracle's numpy code.
__host__ __device__ __forceinline__ uint32_t f32_to_bf16_bits(float f) {
  uint32_t u = f32_bits(f);
  if ((u & 0x7fffffffu) > 0x7f800000u) return (u >> 16) | 0x40u;
  return (u + 0x7fffu + ((u >> 16) & 1u)) >> 16;
}
// fp32 -> int8 of an int8 index (sa_debug_int8_round): round to nearest even, saturate to [-128, 127], NaN -> 0 -- the
// rule of cvt.rni.sat.s8.f32, spelled out so that the host test hook evaluates the very same function.
__host__ __device__ __forceinline__ int f32_to_i8(float f) {
  if (!(f == f)) return 0;
  f = f < -128.f ? -128.f : (f > 127.f ? 127.f : f);
#ifdef __CUDA_ARCH__
  return __float2int_rn(f);
#else
  return static_cast<int>(rintf(f));  // the host's default rounding mode: to nearest even
#endif
}
__device__ __forceinline__ int warp_sum(int v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// Similarity of an index (SA_SIM_* of sa_api.h).  The row term w[r] the scan combines with its accumulator:
//   cosine      1/|c|        0 for an all-zero row (never returned) or a tombstone
//   dotProduct  1            0 for a tombstone (an all-zero row is a live row scoring 0)
//   euclidean   |c|^2 / 2    -1 for a tombstone (an all-zero row is a live row at distance |q|)
// Internally every kernel ranks by a float64 value where larger is better: cosine, <q,c>, and -|q - c|.
constexpr int kSimCos = 0;
constexpr int kSimDot = 1;
constexpr int kSimEuc = 2;
// Element type of an index (SA_ELEM_* of sa_api.h): rows and queries stored as bf16 or as int8.
constexpr int kElemBf16 = 0;
constexpr int kElemI8 = 1;
__host__ __device__ __forceinline__ int elem_bytes(int elem) { return elem == kElemI8 ? 1 : 2; }

// Row term of a row from its float64 sum of squares (dotProduct, euclidean); cosine keeps its fp32 path below.
// |c|^2 is summed in fp64 and rounded once: an fp32 sum of 1536 squares is off by ~1e-4 relative, the size of the whole
// certificate band.  The fp64 sum of squares of bf16 values cannot overflow, so a non-finite sum means a NaN or inf
// element: such a row gets the tombstone term and is never returned, as under cosine and in the definition.
template <int kSim>
__device__ __forceinline__ float row_term_f64(double ss) {
  if (!isfinite(ss)) return kSim == kSimEuc ? -1.0f : 0.0f;
  return kSim == kSimEuc ? __double2float_rn(0.5 * ss) : 1.0f;
}
// An upper bound on the row's norm for Cmax: sqrt in fp64, nudged up, rounded up.  0 (no contribution) for a row that
// row_term_f64 tombstones.
__device__ __forceinline__ unsigned norm_bound_bits(double ss) {
  if (!isfinite(ss)) return 0u;
  return __float_as_uint(__double2float_ru(sqrt(ss) * (1.0 + 0x1p-40)));
}
// Raise the device scalar Cmax (float bits; non-negative floats order like their bits) by the largest bound of a block.
__device__ __forceinline__ void block_raise_cmax(unsigned* cmax, unsigned* blk_max, unsigned mine, bool active) {
  if (threadIdx.x == 0) *blk_max = 0u;
  __syncthreads();
  if (active) atomicMax(blk_max, mine);
  __syncthreads();
  if (threadIdx.x == 0 && *blk_max != 0u) atomicMax(cmax, *blk_max);
}

// inv_norm[r] = 1/sqrt(sum_j row[r][j]^2) over the stored bf16 values, 0 for an all-zero row (cosine).
// One warp per row, 16-byte loads (dim % 8 == 0).
__global__ void sa_rownorm_kernel(const uint16_t* __restrict__ rows, float* __restrict__ inv_norm, long long first,
                                  long long n, int dim) {
  const long long w = (static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (w >= n) return;
  const uint4* src = reinterpret_cast<const uint4*>(rows + (first + w) * dim);
  float ss = 0.f;
  for (int i = lane; i < dim / 8; i += 32) {
    const uint4 x = __ldg(src + i);
    const uint32_t u[4] = {x.x, x.y, x.z, x.w};
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const float a = bf16_bits_to_f32(u[k] & 0xffffu), b = bf16_bits_to_f32(u[k] >> 16);
      ss = fmaf(a, a, ss);
      ss = fmaf(b, b, ss);
    }
  }
  ss = warp_sum(ss);
  if (lane == 0) inv_norm[first + w] = ss > 0.f ? 1.0f / sqrtf(ss) : 0.f;
}

// Square of a bf16 value in fp64: exact, and finite for every finite value (an fp32 square overflows past 2^64).
__device__ __forceinline__ double sq_f64(float a) {
  const double d = static_cast<double>(a);
  return d * d;
}
// fp64 sum of squares of one bf16 row, one warp, every lane gets it.
__device__ __forceinline__ double row_ss_f64(const uint4* __restrict__ src, int nvec, int lane) {
  double ss = 0.0;
  for (int i = lane; i < nvec; i += 32) {
    const uint4 x = __ldg(src + i);
    const uint32_t u[4] = {x.x, x.y, x.z, x.w};
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      ss += sq_f64(bf16_bits_to_f32(u[k] & 0xffffu));
      ss += sq_f64(bf16_bits_to_f32(u[k] >> 16));
    }
  }
  return warp_sum(ss);
}

// dotProduct / euclidean form of sa_rownorm_kernel: w[r] = row_term_f64 of the row, and Cmax raised to cover it.
// first < 0: recompute Cmax only (sa_corpus_bind), leaving w untouched.  One warp per row.
template <int kSim>
__global__ void sa_rowterm_kernel(const uint16_t* __restrict__ rows, float* __restrict__ w_out, long long first,
                                  long long n, int dim, unsigned* __restrict__ cmax) {
  __shared__ unsigned blk_max;
  const long long w = (static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  const bool active = w < n;
  unsigned nb = 0u;
  if (active) {
    const long long r = (first < 0 ? 0 : first) + w;
    const double ss = row_ss_f64(reinterpret_cast<const uint4*>(rows + r * dim), dim / 8, lane);
    if (lane == 0 && first >= 0) w_out[r] = row_term_f64<kSim>(ss);
    nb = norm_bound_bits(ss);
  }
  block_raise_cmax(cmax, &blk_max, nb, active && lane == 0);
}

// dst_bf16[r][:] = RNE(src_f32[r][:]); optionally also inv_norm[r] (corpus ingest, cosine).  One warp per row.
__global__ void sa_convert_rows_kernel(const float* __restrict__ src, uint16_t* __restrict__ dst,
                                       float* __restrict__ inv_norm, long long n, int dim) {
  const long long w = (static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (w >= n) return;
  const float4* s = reinterpret_cast<const float4*>(src + w * dim);
  uint2* d = reinterpret_cast<uint2*>(dst + w * dim);
  float ss = 0.f;
  for (int i = lane; i < dim / 4; i += 32) {
    const float4 x = __ldg(s + i);
    const uint32_t b0 = f32_to_bf16_bits(x.x), b1 = f32_to_bf16_bits(x.y), b2 = f32_to_bf16_bits(x.z),
                   b3 = f32_to_bf16_bits(x.w);
    d[i] = make_uint2(b0 | (b1 << 16), b2 | (b3 << 16));
    const float r0 = bf16_bits_to_f32(b0), r1 = bf16_bits_to_f32(b1), r2 = bf16_bits_to_f32(b2),
                r3 = bf16_bits_to_f32(b3);
    ss = fmaf(r0, r0, ss);
    ss = fmaf(r1, r1, ss);
    ss = fmaf(r2, r2, ss);
    ss = fmaf(r3, r3, ss);
  }
  if (inv_norm != nullptr) {
    ss = warp_sum(ss);
    if (lane == 0) inv_norm[w] = ss > 0.f ? 1.0f / sqrtf(ss) : 0.f;
  }
}

// dotProduct / euclidean corpus ingest: dst_bf16[r][:] = RNE(src_f32[r][:]), w[r] = row_term_f64, Cmax raised.
template <int kSim>
__global__ void sa_convert_rows_term_kernel(const float* __restrict__ src, uint16_t* __restrict__ dst,
                                            float* __restrict__ w_out, long long n, int dim, unsigned* __restrict__ cmax) {
  __shared__ unsigned blk_max;
  const long long w = (static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  const bool active = w < n;
  unsigned nb = 0u;
  if (active) {
    const float4* s = reinterpret_cast<const float4*>(src + w * dim);
    uint2* d = reinterpret_cast<uint2*>(dst + w * dim);
    double ss = 0.0;
    for (int i = lane; i < dim / 4; i += 32) {
      const float4 x = __ldg(s + i);
      const uint32_t b0 = f32_to_bf16_bits(x.x), b1 = f32_to_bf16_bits(x.y), b2 = f32_to_bf16_bits(x.z),
                     b3 = f32_to_bf16_bits(x.w);
      d[i] = make_uint2(b0 | (b1 << 16), b2 | (b3 << 16));
      const float r0 = bf16_bits_to_f32(b0), r1 = bf16_bits_to_f32(b1), r2 = bf16_bits_to_f32(b2),
                  r3 = bf16_bits_to_f32(b3);
      ss += sq_f64(r0);
      ss += sq_f64(r1);
      ss += sq_f64(r2);
      ss += sq_f64(r3);
    }
    ss = warp_sum(ss);
    if (lane == 0) w_out[w] = row_term_f64<kSim>(ss);
    nb = norm_bound_bits(ss);
  }
  block_raise_cmax(cmax, &blk_max, nb, active && lane == 0);
}

// ---- int8 rows.  Sums of int8 products are exact integers (|sum| <= dim 2^14 <= 2^30 for dim <= 65536), so the sum of
// squares is exact, and each row term is rounded once from it in fp64: 1/|c| (0 for an all-zero row), 1, or |c|^2/2.
__device__ __forceinline__ int dp4a_s8(unsigned a, unsigned b, int c) {
  return __dp4a(static_cast<int>(a), static_cast<int>(b), c);
}
__device__ __forceinline__ float row_term_i8(int sim, int ss) {
  const double d = static_cast<double>(ss);
  if (sim == kSimCos) return ss > 0 ? __double2float_rn(1.0 / sqrt(d)) : 0.f;
  return sim == kSimEuc ? __double2float_rn(0.5 * d) : 1.0f;
}
// Exact sum of squares of one int8 row, one warp (16-byte loads, dim % 128 == 0), every lane gets it.
__device__ __forceinline__ int row_ss_i8(const uint4* __restrict__ src, int nvec, int lane) {
  int ss = 0;
  for (int i = lane; i < nvec; i += 32) {
    const uint4 x = __ldg(src + i);
    ss = dp4a_s8(x.x, x.x, ss);
    ss = dp4a_s8(x.y, x.y, ss);
    ss = dp4a_s8(x.z, x.z, ss);
    ss = dp4a_s8(x.w, x.w, ss);
  }
  return warp_sum(ss);
}

// Row terms of int8 rows written in place (sa_corpus_commit), Cmax raised to cover them.  first < 0: recompute Cmax only
// (sa_corpus_bind), leaving w untouched.  One warp per row.
__global__ void sa_rowterm_i8_kernel(const int8_t* __restrict__ rows, float* __restrict__ w_out, long long first,
                                     long long n, int dim, int sim, unsigned* __restrict__ cmax) {
  __shared__ unsigned blk_max;
  const long long w = (static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  const bool active = w < n;
  unsigned nb = 0u;
  if (active) {
    const long long r = (first < 0 ? 0 : first) + w;
    const int ss = row_ss_i8(reinterpret_cast<const uint4*>(rows + r * dim), dim / 16, lane);
    if (lane == 0 && first >= 0) w_out[r] = row_term_i8(sim, ss);
    nb = norm_bound_bits(static_cast<double>(ss));
  }
  block_raise_cmax(cmax, &blk_max, nb, active && lane == 0);
}

// dst_i8[r][:] = f32_to_i8(src_f32[r][:]).  Rows (w_out != nullptr): also the row term and Cmax, as
// sa_rowterm_i8_kernel; queries (w_out == nullptr): the conversion only.  One warp per row, 16-byte loads.
__global__ void sa_convert_rows_i8_kernel(const float* __restrict__ src, int8_t* __restrict__ dst, float* __restrict__ w_out,
                                          long long n, int dim, int sim, unsigned* __restrict__ cmax) {
  __shared__ unsigned blk_max;
  const long long w = (static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  const bool active = w < n;
  unsigned nb = 0u;
  if (active) {
    const float4* s = reinterpret_cast<const float4*>(src + w * dim);
    unsigned* d = reinterpret_cast<unsigned*>(dst + w * dim);
    int ss = 0;
    for (int i = lane; i < dim / 4; i += 32) {
      const float4 x = __ldg(s + i);
      const unsigned b = (static_cast<unsigned>(f32_to_i8(x.x)) & 0xffu) |
                         ((static_cast<unsigned>(f32_to_i8(x.y)) & 0xffu) << 8) |
                         ((static_cast<unsigned>(f32_to_i8(x.z)) & 0xffu) << 16) |
                         (static_cast<unsigned>(f32_to_i8(x.w)) << 24);
      d[i] = b;
      ss = dp4a_s8(b, b, ss);
    }
    ss = warp_sum(ss);
    if (w_out != nullptr) {
      if (lane == 0) w_out[w] = row_term_i8(sim, ss);
      nb = norm_bound_bits(static_cast<double>(ss));
    }
  }
  if (w_out != nullptr) block_raise_cmax(cmax, &blk_max, nb, active && lane == 0);  // w_out is uniform over the grid
}

// Per-query filter over the rows' 64-bit tags (sa_filter of sa_api.h, same layout).  One definition of the predicate
// serves the scan's epilogue, the exact fallback scan and the host test hook (sa_debug_filter_pass).
struct Filter {
  unsigned long long all_of;     // every bit must be set on the row
  unsigned long long none_of;    // no bit may be set
  unsigned long long any_of[2];  // each nonzero word: at least one of its bits must be set
};
__host__ __device__ __forceinline__ bool filter_pass(unsigned long long t, const Filter& f) {
  return ((t & f.all_of) == f.all_of) & ((t & f.none_of) == 0ull) & ((f.any_of[0] == 0ull) | ((t & f.any_of[0]) != 0ull)) &
         ((f.any_of[1] == 0ull) | ((t & f.any_of[1]) != 0ull));
}

// Order-preserving map: (score desc, row asc)  <=>  key desc.  The high word is float_to_key(score).
__host__ __device__ __forceinline__ unsigned long long make_key(float s, int row) {
  return (static_cast<unsigned long long>(float_to_key(s)) << 32) | static_cast<uint32_t>(~static_cast<uint32_t>(row));
}
__host__ __device__ __forceinline__ int key_row(unsigned long long k) { return static_cast<int>(~static_cast<uint32_t>(k)); }

// ------------------------------------------------------------------------------------------------------------------
// Stage 2 of the search: merge the per-lane candidate lists of one query, certify, re-score exactly.
//
// Notation (all in the scan's "approximate units": a(r) = fp32_accumulate(q . c_r) * fl(w_r) (euclidean: - fl(w_r)), no
// 1/|q| factor; the exact value in the same units is e(r) = <q, c_r> / |c_r| = cos(q, c_r) * |q| for cosine, <q, c_r>
// for dotProduct, <q, c_r> - |c_r|^2 / 2 = (|q|^2 - |q - c_r|^2) / 2 for euclidean):
//   eps     bound on |a(r) - e(r)|, cert_eps below (eps_rel from the engine: ~dim * 2^-23, DESIGN.md section 4.2)
//   U       union of the TL lane lists of the query;  drop_l >= a(r) for every row r of lane l that is not in U
//   A_k     k-th largest a over U
// Claim.  Let band = A_k - 2 eps.  If drop_l < band for every lane l, then every row outside U has a < band, A_k is the
// k-th largest a over the WHOLE corpus, and every row of the exact top-k has a >= T - eps >= A_k - 2 eps = band (T = k-th
// largest e; T >= A_k - eps because the k rows with a >= A_k have e >= A_k - eps).  So the exact top-k is contained in
// {r in U : a(r) >= band}; re-scoring that set in float64 and sorting by (value desc, row asc) IS the brute-force answer.
// A lane with drop_l >= band ("ambiguous") may have discarded such a row: the query then gets one work item per ambiguous
// lane for the exact fallback scan (sa_fixup_kernel), which re-reads only those lanes' tiles.
// ------------------------------------------------------------------------------------------------------------------
struct FixEntry {
  int q;        // query index within the whole search
  int lane_tl;  // tile lane | (tile lanes of that scan launch << 16)
};
struct FixQuery {
  double qq;    // |q|^2
  float eps;    // the certificate's bound |a - e| for this query (cert_eps)
  float band;   // prefilter threshold in approximate units (-inf: everything is re-scored)
  int lock;     // spin lock of the query's result list during the fallback scan (0 = free)
};

struct MergeParams {
  const float* part_score;  // [grid CTAs][128][kKL] from the scan
  const int* part_idx;
  const float* part_drop;   // [grid CTAs][128]
  const void* corpus;       // [capacity][dim] bf16 or int8 (elem)
  const void* queries;      // [nq][dim] bf16 or int8 (this launch's queries)
  int dim;
  int nq;
  int k;
  int cg;                   // CTAs per unit in the scan that produced the lists
  int nqb;
  int tl_count;
  int unit_map;             // same mapping switch as ScanParams::unit_map
  int q0;                   // index of this launch's first query within the whole search
  float eps_rel;            // relative accumulation bound of the scan (cert_eps)
  int sim;                  // kSimCos / kSimDot / kSimEuc
  int elem;                 // kElemBf16 / kElemI8
  const unsigned* cmax;     // device scalar (float bits): upper bound on |c| over the committed rows (not cosine)
  double* res64;            // [nq][k] this launch's slice of the search's internal result: value (float64) ...
  int* residx;              // ... and shard-local row, -1 / -inf when fewer than k rows qualify
  FixEntry* fix_entries;    // work queue of the fallback scan
  int* fix_count;           // zero at the start of a search
  FixQuery* fix_query;      // [search nq]
  int force_fix;            // test hook: 1 = treat every lane as ambiguous (the fallback then recomputes everything)
  unsigned* bound_out;      // sampling pre-pass only (else nullptr): publish each query's max(k, kKL)-th best score of the
                            // sample into the scan's shared thresholds [nq] and do nothing else
};

constexpr int kMergeThreads = 160;  // >= kMaxLanes: one thread per tile lane in the head tournament
constexpr int kMergeWarps = kMergeThreads / 32;
constexpr int kMaxLanes = 132;      // tile lanes of one scan launch (the planner caps TL here): one per H100 SM
constexpr int kSelMax = 128;        // candidates re-scored per query without the fallback

__device__ __forceinline__ float key_score(unsigned long long k) {
  return key_to_float(static_cast<unsigned>(k >> 32));
}

// The internal value from the exact sums <q,c>, |c|^2 and |q|^2 (the one formula of every element type).
__device__ __forceinline__ double exact_value_from_sums(double dot, double dd, double qq, int sim) {
  if (sim == kSimDot) return dot;
  if (sim == kSimEuc) {
    const double d2 = __dadd_rn(__dsub_rn(qq, 2.0 * dot), dd);  // no contraction: the oracle evaluates the same two ops
    return -sqrt(d2 > 0.0 ? d2 : 0.0);
  }
  const double den = qq * dd;
  return den > 0.0 ? dot / sqrt(den) : 0.0;
}

// Exact internal value of (query, corpus row), one warp: bf16 x bf16 products are exact in fp32; sums of products and of
// squares in float64, lane-strided then a butterfly.  Every lane returns the same value.  Used by the merge kernel AND
// the fallback scan, so the two produce bit-identical values for the same pair.  Larger is better:
//   cosine      <q,c> / sqrt(|q|^2 |c|^2)   (0 when either is all-zero)
//   dotProduct  <q,c>
//   euclidean   -sqrt(max(d2, 0)),  d2 = (|q|^2 - 2 <q,c>) + |c|^2   -- one fixed formula, the oracle's too
// int8 (elem == kElemI8): the sums are exact int32 sums (dp4a), converted to float64 exactly; the formulas are the same.
// nvec = 16-byte vectors per row (dim / 8 bf16, dim / 16 int8).
__device__ __forceinline__ double exact_value_warp(const uint4* __restrict__ qv, const uint4* __restrict__ cv, int nvec,
                                                   double qq, int lane, int sim, int elem) {
  double dot = 0.0, dd = 0.0;
  if (elem == kElemI8) {
    int idot = 0, idd = 0;
    for (int i = lane; i < nvec; i += 32) {
      const uint4 x = __ldg(qv + i);
      const uint4 y = __ldg(cv + i);
      idot = dp4a_s8(x.x, y.x, dp4a_s8(x.y, y.y, dp4a_s8(x.z, y.z, dp4a_s8(x.w, y.w, idot))));
      idd = dp4a_s8(y.x, y.x, dp4a_s8(y.y, y.y, dp4a_s8(y.z, y.z, dp4a_s8(y.w, y.w, idd))));
    }
    dot = static_cast<double>(warp_sum(idot));
    dd = static_cast<double>(warp_sum(idd));
    return exact_value_from_sums(dot, dd, qq, sim);
  }
  for (int i = lane; i < nvec; i += 32) {
    const uint4 x = __ldg(qv + i);
    const uint4 y = __ldg(cv + i);
    const uint32_t u[4] = {x.x, x.y, x.z, x.w};
    const uint32_t v[4] = {y.x, y.y, y.z, y.w};
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const float a0 = bf16_bits_to_f32(u[k] & 0xffffu), a1 = bf16_bits_to_f32(u[k] >> 16);
      const float b0 = bf16_bits_to_f32(v[k] & 0xffffu), b1 = bf16_bits_to_f32(v[k] >> 16);
      dot += static_cast<double>(a0 * b0);
      dot += static_cast<double>(a1 * b1);
      dd += static_cast<double>(b0 * b0);
      dd += static_cast<double>(b1 * b1);
    }
  }
  dot = warp_sum(dot);
  if (sim == kSimDot) return dot;
  dd = warp_sum(dd);
  return exact_value_from_sums(dot, dd, qq, sim);
}

// The certificate's bound eps >= |a(r) - e(r)| for every committed row r, rounded up (DESIGN.md section 4.2).
//   cosine      eps_rel |q|                                    (the row's norm cancels against w = 1/|c|)
//   dotProduct  eps_rel |q| Cmax                               (|acc - <q,c>| <= dim 2^-23 |q| |c|)
//   euclidean   (eps_rel + 2^-23) |q| Cmax + 2^-23 Cmax^2 + 2^-50 |q|^2
//               (accumulation as above; w rounded once from fp64: 2^-24 |c|^2/2; the subtraction: 2^-24 (|acc| + w);
//                the last term covers the fallback's fp64 conversion of a distance into these units)
// Cmax is an upper bound on the committed rows' norms, kept on the device: reading it costs the search no host sync.
__device__ __forceinline__ float cert_eps(int sim, double qq, float eps_rel, const unsigned* cmax) {
  const double qn = sqrt(qq);
  if (sim == kSimCos) return __double2float_ru(qn * static_cast<double>(eps_rel));
  const double cm = static_cast<double>(__uint_as_float(*cmax));
  if (sim == kSimDot) return __double2float_ru(qn * cm * static_cast<double>(eps_rel) * (1.0 + 0x1p-40));
  const double u = 0x1p-23;
  return __double2float_ru(((static_cast<double>(eps_rel) + u) * qn * cm + u * cm * cm + 0x1p-50 * qq) * (1.0 + 0x1p-40));
}

// An exact internal value (exact_value_warp) in the scan's units, rounded down (towards a wider prefilter).
__device__ __forceinline__ float value_to_scan_rd(int sim, double v, double qq) {
  if (sim == kSimCos) return __double2float_rd(v * sqrt(qq));
  if (sim == kSimDot) return __double2float_rd(v);
  return __double2float_rd(0.5 * (qq - v * v));  // v = -d: (|q|^2 - d^2) / 2
}
__device__ __forceinline__ double query_norm2_warp(const uint4* __restrict__ qv, int nvec, int lane, int elem) {
  if (elem == kElemI8) return static_cast<double>(row_ss_i8(qv, nvec, lane));  // exact
  double qq = 0.0;
  for (int i = lane; i < nvec; i += 32) {
    const uint4 x = __ldg(qv + i);
    const uint32_t u[4] = {x.x, x.y, x.z, x.w};
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const float a = bf16_bits_to_f32(u[k] & 0xffffu), b = bf16_bits_to_f32(u[k] >> 16);
      qq += static_cast<double>(a * a);
      qq += static_cast<double>(b * b);
    }
  }
  return warp_sum(qq);
}

// (value desc, row asc): does (c1, r1) come before (c2, r2)?
__host__ __device__ __forceinline__ bool result_before(double c1, int r1, double c2, int r2) {
  return c1 > c2 || (c1 == c2 && r1 < r2);
}

// One block per query.
template <int kKL>
__global__ void __launch_bounds__(kMergeThreads) sa_merge_rescore_kernel(const MergeParams p) {
  __shared__ unsigned long long keys[kMaxLanes * kKL];
  __shared__ unsigned long long sel[kSelMax];
  __shared__ double cs[kSelMax];
  __shared__ unsigned long long wbest[2][kMergeWarps];
  __shared__ double qq_s;
  __shared__ int nsel_s;
  __shared__ int namb_s;

  const int q = blockIdx.x;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int rows_per_unit = 128 * p.cg;
  const int qb = q / rows_per_unit;
  const int r = q % rows_per_unit;
  const int cta_in_unit = r / 128, row = r % 128;
  const int TL = p.tl_count;
  const int ncand = TL * kKL;
  auto cta_of_lane = [&](int tl) -> size_t {
    const int unit = p.unit_map == 0 ? tl * p.nqb + qb : qb * TL + tl;
    return static_cast<size_t>(unit) * p.cg + cta_in_unit;
  };

  for (int i = tid; i < ncand; i += kMergeThreads) {
    const int tl = i / kKL, e = i % kKL;
    const size_t o = (cta_of_lane(tl) * 128 + row) * kKL + e;
    keys[i] = make_key(p.part_score[o], p.part_idx[o]);
  }
  float my_drop = -INFINITY;
  if (tid < TL) my_drop = p.part_drop[cta_of_lane(tid) * 128 + row];
  if (tid == 0) {
    nsel_s = 0;
    namb_s = 0;
  }
  const size_t row_bytes = static_cast<size_t>(p.dim) * elem_bytes(p.elem);
  const uint4* qv = reinterpret_cast<const uint4*>(static_cast<const char*>(p.queries) + q * row_bytes);
  const int nvec = static_cast<int>(row_bytes / 16);
  if (warp == kMergeWarps - 1) {
    const double qq = query_norm2_warp(qv, nvec, lane, p.elem);
    if (lane == 0) qq_s = qq;
  }
  __syncthreads();

  // ---- A_k: k rounds of arg-max over the heads of the (sorted) lane lists; thread t owns lane t.  k may exceed kKL (a
  // deep search): a lane then runs out of entries (cand 0) and the others supply the remaining rounds.
  int head = 0;
  unsigned long long kth = 0;  // key of the k-th best candidate, 0 if fewer than k exist
  const int rounds = p.bound_out != nullptr ? (p.k > kKL ? p.k : kKL) : p.k;
  for (int round = 0; round < rounds; ++round) {
    const unsigned long long cand = (tid < TL && head < kKL) ? keys[tid * kKL + head] : 0ull;
    unsigned long long wb = cand;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const unsigned long long other = __shfl_xor_sync(0xffffffffu, wb, o);
      wb = other > wb ? other : wb;
    }
    if (lane == 0) wbest[round & 1][warp] = wb;
    __syncthreads();
    unsigned long long gb = wbest[round & 1][0];
#pragma unroll
    for (int w = 1; w < kMergeWarps; ++w) gb = wbest[round & 1][w] > gb ? wbest[round & 1][w] : gb;
    if (gb == 0ull || key_row(gb) < 0) {  // only empty slots remain: fewer than k candidates
      kth = 0;
      break;
    }
    if (cand == gb) ++head;  // keys of real candidates are unique (rows are unique per query)
    kth = gb;
  }
  if (p.bound_out != nullptr) {
    // Sampling pre-pass: at least kKL rows of the corpus score >= the sample's kKL-th best, so no row scoring less can be
    // in this query's global top-kKL: a valid shared threshold for the full scan that follows (kth >> 32 is the score's
    // float_to_key, the scan's own key: see make_key).
    // A deep search (k > kKL) publishes the sample's k-th best over the union instead, a bound on the global k-th best;
    // a union of fewer than k rows publishes nothing.
    if (tid == 0 && kth != 0ull) atomicMax(p.bound_out + q, static_cast<unsigned>(kth >> 32));
    return;
  }
  const double qq = qq_s;
  // eps and band, rounded towards "wider"
  const float eps = cert_eps(p.sim, qq, p.eps_rel, p.cmax);
  const float band = (kth != 0ull) ? __fsub_rd(key_score(kth), __fmul_ru(2.0f, eps)) : -INFINITY;

  // ---- ambiguous lanes, and the band candidates of U
  const bool amb = p.force_fix ? (tid < TL) : (tid < TL && my_drop > -INFINITY && my_drop >= band);
  if (amb) atomicAdd(&namb_s, 1);
  if (tid < TL) {
    for (int e = 0; e < kKL; ++e) {
      const unsigned long long kk = keys[tid * kKL + e];
      if (key_row(kk) < 0 || !(key_score(kk) >= band)) break;  // lists are sorted: nothing further qualifies
      const int pos = atomicAdd(&nsel_s, 1);
      if (pos < kSelMax) sel[pos] = kk;
    }
  }
  __syncthreads();
  const bool overflow = nsel_s > kSelMax;  // more band candidates than we re-score here: every lane goes to the fallback
  const int nsel = min(nsel_s, kSelMax);

  // ---- exact re-scoring: warp w takes candidates w, w + kMergeWarps, ...
  for (int c = warp; c < nsel; c += kMergeWarps) {
    const int crow = key_row(sel[c]);
    const uint4* cv = reinterpret_cast<const uint4*>(static_cast<const char*>(p.corpus) + crow * row_bytes);
    const double v = exact_value_warp(qv, cv, nvec, qq, lane, p.sim, p.elem);
    if (lane == 0) cs[c] = v;
  }
  __syncthreads();

  // ---- rank by counting; the first k go to the result
  for (int i = tid; i < max(nsel, p.k); i += kMergeThreads) {
    if (i < nsel) {
      const double ci = cs[i];
      const int ri = key_row(sel[i]);
      int rank = 0;
      for (int j = 0; j < nsel; ++j) rank += result_before(cs[j], key_row(sel[j]), ci, ri) ? 1 : 0;
      if (rank < p.k) {
        p.res64[static_cast<size_t>(q) * p.k + rank] = ci;
        p.residx[static_cast<size_t>(q) * p.k + rank] = ri;
      }
    }
    if (i >= nsel && i < p.k) {  // nsel >= min(k, eligible rows)
      p.res64[static_cast<size_t>(q) * p.k + i] = -INFINITY;
      p.residx[static_cast<size_t>(q) * p.k + i] = -1;
    }
  }

  // ---- work items for the fallback scan
  if (namb_s > 0 || overflow) {
    if (tid < TL && (amb || overflow)) {
      const int pos = atomicAdd(p.fix_count, 1);
      p.fix_entries[pos].q = p.q0 + q;
      p.fix_entries[pos].lane_tl = tid | (TL << 16);
    }
    if (tid == 0) {
      FixQuery fq;
      fq.qq = qq;
      fq.eps = eps;
      fq.band = band;
      fq.lock = 0;
      p.fix_query[p.q0 + q] = fq;
    }
  }
}

// ------------------------------------------------------------------------------------------------------------------
// Stage 3: exact fallback scan of the ambiguous (query, lane) pairs + finalisation of the search's outputs.
// Always launched; with an empty work queue (the normal case) it only converts the internal result to the caller's
// output arrays and re-zeroes the scan's scratch for the next search.
//
// Work item = (queue entry, chunk of kFixChunkTiles tiles of that lane).  A CTA stages the query's bytes in shared memory;
// each warp walks rows: fp32 dot (CUDA cores) * w (euclidean: - w) -> a'(r), whose error is inside eps; rows with a' >=
// max(band, current k-th exact value in approximate units - eps) are re-scored exactly and inserted into the WARP's own list (no
// sharing between warps, so no locks in shared memory); at the end of the item one thread folds the warps' lists into the
// query's result under the query's lock (rows already present are skipped).  The last CTA to finish finalises.
// ------------------------------------------------------------------------------------------------------------------
struct PackedHit {
  double score;       // the returned value, float64: cosine, dot product or Euclidean distance
  long long row;      // global row (shard offset applied), -1 = none
};

struct FixParams {
  const FixEntry* entries;
  int* fix_count;
  int* done_count;
  FixQuery* fix_query;
  const void* corpus;       // bf16 or int8 (elem)
  const float* row_term;
  const void* queries;      // [nq][dim] the whole search
  long long n_rows;
  int num_tiles;
  int dim;
  int nq;
  int k;
  int chunks_per_entry;     // ceil(max tiles per lane / kFixChunkTiles)
  int sim;                  // kSimCos / kSimDot / kSimEuc
  int elem;                 // kElemBf16 / kElemI8
  double* res64;            // [nq][k] internal result (read / updated here)
  int* residx;
  // finalisation: the internal value becomes the returned one (euclidean: the distance, -v)
  float* out_score;         // [nq][k] fp32 value
  int* out_idx;             // [nq][k] shard-local row
  double* out_score64;      // optional
  PackedHit* out_packed;    // optional: (cosine f64, global row) for the cross-shard exchange
  long long row_offset;     // first global row of this shard
  unsigned* zero_a;         // scratch to re-zero for the next search (shared thresholds) ...
  int zero_a_n;
  int* zero_b;              // ... drift counters
  int zero_b_n;
  unsigned* zero_c;         // ... and the lanes' second-best table (window bound)
  int zero_c_n;
  const unsigned long long* row_tags;  // filtered search: [capacity] the rows' tags ...
  const Filter* filters;               // ... and [nq] the queries' filters; nullptr: unfiltered
};

constexpr int kFixThreads = 256;
constexpr int kFixChunkTiles = 8;
constexpr int kFixMaxK = 64;  // per-warp lists of k <= 64 entries in shared memory (SA_MAX_K)
constexpr int kFixSmemMax = 2 * 65536;  // dynamic shared memory: one bf16 query row of SA_MAX_DIM elements

__device__ __forceinline__ void fix_finalize(const FixParams& p, int first, int stride) {
  const int total = p.nq * p.k;
  for (int i = first; i < total; i += stride) {
    const double s = p.sim == kSimEuc ? -p.res64[i] : p.res64[i];  // empty slots: -inf -> +inf for distances
    const int r = p.residx[i];
    p.out_score[i] = static_cast<float>(s);
    p.out_idx[i] = r;
    if (p.out_score64 != nullptr) p.out_score64[i] = s;
    if (p.out_packed != nullptr) {
      PackedHit h;
      h.score = s;
      h.row = r >= 0 ? static_cast<long long>(r) + p.row_offset : -1ll;
      p.out_packed[i] = h;
    }
  }
  for (int i = first; i < p.zero_a_n; i += stride) p.zero_a[i] = 0u;
  for (int i = first; i < p.zero_b_n; i += stride) p.zero_b[i] = 0;
  for (int i = first; i < p.zero_c_n; i += stride) p.zero_c[i] = 0u;
}

// Sorted insertion of (c, r) into a (cosine desc, row asc) list of k slots (row -1 = empty); skips a row already present.
template <typename D, typename I>
__device__ __forceinline__ void fix_list_insert(D* cosv, I* rowv, int k, double c, int r) {
  int pos = k;
  for (int i = 0; i < k; ++i) {
    const int ri = rowv[i];
    if (ri == r) return;
    if (pos == k && (ri < 0 || result_before(c, r, cosv[i], ri))) pos = i;
  }
  if (pos == k) return;
  for (int i = k - 1; i > pos; --i) {
    cosv[i] = cosv[i - 1];
    rowv[i] = rowv[i - 1];
  }
  cosv[pos] = c;
  rowv[pos] = r;
}

__global__ void __launch_bounds__(kFixThreads) sa_fixup_kernel(const FixParams p) {
  extern __shared__ uint4 q_s[];  // the query's row bytes as they are (bf16 or int8): at most 2 SA_MAX_DIM bytes
  constexpr int kWarps = kFixThreads / 32;
  __shared__ double l_cos[kWarps][kFixMaxK];  // one list per warp, touched by that warp's lane 0 only
  __shared__ int l_row[kWarps][kFixMaxK];
  __shared__ float thr0_s;
  __shared__ int last_s;

  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int count = *reinterpret_cast<volatile int*>(p.fix_count);
  if (count == 0) {  // nothing was ambiguous: the internal result is final
    fix_finalize(p, blockIdx.x * kFixThreads + tid, gridDim.x * kFixThreads);
    return;
  }

  const bool i8 = p.elem == kElemI8;
  const size_t row_bytes = static_cast<size_t>(p.dim) * elem_bytes(p.elem);
  const int nvec = static_cast<int>(row_bytes / 16);
  const long long items = static_cast<long long>(count) * p.chunks_per_entry;
  for (long long item = blockIdx.x; item < items; item += gridDim.x) {
    const FixEntry en = p.entries[item / p.chunks_per_entry];
    const int chunk = static_cast<int>(item % p.chunks_per_entry);
    const int tl = en.lane_tl & 0xffff, TL = en.lane_tl >> 16;
    const int t_first = tl + chunk * kFixChunkTiles * TL;
    if (t_first >= p.num_tiles) continue;  // block-uniform
    FixQuery* fq = p.fix_query + en.q;
    const double qq = fq->qq;
    const float eps = fq->eps;
    volatile double* g_cos = p.res64 + static_cast<size_t>(en.q) * p.k;
    volatile int* g_row = p.residx + static_cast<size_t>(en.q) * p.k;
    const uint4* qv = reinterpret_cast<const uint4*>(static_cast<const char*>(p.queries) + en.q * row_bytes);
    Filter flt = {0ull, 0ull, {0ull, 0ull}};  // match-all unless the search is filtered
    if (p.filters != nullptr) flt = p.filters[en.q];

    __syncthreads();  // previous item's smem no longer in use
    for (int i = tid; i < nvec; i += kFixThreads) q_s[i] = __ldg(qv + i);
    for (int i = tid; i < kWarps * kFixMaxK; i += kFixThreads) {
      l_cos[i / kFixMaxK][i % kFixMaxK] = -INFINITY;
      l_row[i / kFixMaxK][i % kFixMaxK] = -1;
    }
    if (tid == 0) {
      // prefilter threshold: the band of the merge kernel, tightened by the k-th exact value found so far
      float thr = fq->band;
      const int rk = g_row[p.k - 1];
      if (rk >= 0) thr = fmaxf(thr, __fsub_rd(value_to_scan_rd(p.sim, g_cos[p.k - 1], qq), eps));
      thr0_s = thr;
    }
    __syncthreads();
    float thr = thr0_s;           // per warp from here on: tightened by the warp's own list (uniform across its lanes)
    double* wc = l_cos[warp];
    int* wrow = l_row[warp];

    for (int ti = 0; ti < kFixChunkTiles; ++ti) {
      const int t = t_first + ti * TL;
      if (t >= p.num_tiles) break;
      for (int rr = warp; rr < 256; rr += kWarps) {
        const long long r = static_cast<long long>(t) * 256 + rr;
        if (r >= p.n_rows) break;
        const float wr = __ldg(p.row_term + r);
        if (p.sim == kSimEuc ? !(wr >= 0.f) : !(wr > 0.f)) continue;  // rows that are not live are never returned
        if (p.filters != nullptr && !filter_pass(__ldg(p.row_tags + r), flt)) continue;  // nor rows the filter excludes
        const uint4* cv = reinterpret_cast<const uint4*>(static_cast<const char*>(p.corpus) + r * row_bytes);
        float acc;
        if (i8) {
          // exact int32 dot (dp4a), rounded once to fp32: the scan's accumulator exactly, so a' below is the scan's a
          int iacc = 0;
          for (int i = lane; i < nvec; i += 32) {
            const uint4 y = __ldg(cv + i);
            const uint4 x = q_s[i];
            iacc = dp4a_s8(x.x, y.x, dp4a_s8(x.y, y.y, dp4a_s8(x.z, y.z, dp4a_s8(x.w, y.w, iacc))));
          }
          acc = __int2float_rn(warp_sum(iacc));
        } else {
          // both operands widened from their bits (bf16 -> fp32 is exact)
          acc = 0.f;
          for (int i = lane; i < nvec; i += 32) {
            const uint4 y = __ldg(cv + i);
            const uint4 x = q_s[i];
            const uint32_t u[4] = {x.x, x.y, x.z, x.w};
            const uint32_t v[4] = {y.x, y.y, y.z, y.w};
#pragma unroll
            for (int k = 0; k < 4; ++k) {
              acc = fmaf(bf16_bits_to_f32(u[k] & 0xffffu), bf16_bits_to_f32(v[k] & 0xffffu), acc);
              acc = fmaf(bf16_bits_to_f32(u[k] >> 16), bf16_bits_to_f32(v[k] >> 16), acc);
            }
          }
          acc = warp_sum(acc);
        }
        const float ap = p.sim == kSimEuc ? acc - wr : acc * wr;
        if (!(ap >= thr)) continue;  // warp-uniform (every lane holds the same sum)
        const double c = exact_value_warp(qv, cv, nvec, qq, lane, p.sim, p.elem);
        float nt = thr;
        if (lane == 0) {
          fix_list_insert(wc, wrow, p.k, c, static_cast<int>(r));
          if (wrow[p.k - 1] >= 0) nt = fmaxf(thr, __fsub_rd(value_to_scan_rd(p.sim, wc[p.k - 1], qq), eps));
        }
        thr = __shfl_sync(0xffffffffu, nt, 0);
      }
    }
    __syncthreads();
    if (tid == 0) {  // fold the warps' lists into the query's result under its lock (rows already present are skipped)
      bool any = false;
      for (int w = 0; w < kWarps; ++w) any = any || l_row[w][0] >= 0;
      if (any) {
        while (atomicCAS(&fq->lock, 0, 1) != 0) {
        }
        __threadfence();
        for (int w = 0; w < kWarps; ++w)
          for (int i = 0; i < p.k && l_row[w][i] >= 0; ++i) fix_list_insert(g_cos, g_row, p.k, l_cos[w][i], l_row[w][i]);
        __threadfence();
        atomicExch(&fq->lock, 0);
      }
    }
  }

  // ---- the last CTA to get here finalises (every result list is complete by then)
  __syncthreads();
  if (tid == 0) {
    __threadfence();
    last_s = (atomicAdd(p.done_count, 1) == static_cast<int>(gridDim.x) - 1) ? 1 : 0;
  }
  __syncthreads();
  if (last_s) {
    __threadfence();
    fix_finalize(p, tid, kFixThreads);
    if (tid == 0) {
      *p.fix_count = 0;
      *p.done_count = 0;
    }
  }
}

// After the all-gather of the packed per-shard results: per query, merge G shard lists of k (already sorted, global
// rows) into the global top-k by (value desc, global row asc); asc = 1 (distances): by (value asc, global row asc).
// The scores are negated on load and back on store when asc, so one "larger is better" loop serves both.  One warp per query, lane g holds the head of shard g's
// list (G <= 32): k rounds of a warp arg-max, the winning lane advances.  The lists are first staged in shared memory
// with coalesced 16-byte loads.
constexpr int kMergePackedWarps = 4;
constexpr int kMergePackedMaxK = 32;
__global__ void __launch_bounds__(kMergePackedWarps * 32)
sa_merge_packed_kernel(const PackedHit* __restrict__ hits, int n_shards, int nq, int k, float* __restrict__ out_score,
                       long long* __restrict__ out_idx, int asc) {
  __shared__ PackedHit stage[kMergePackedWarps][32 * kMergePackedMaxK / 4];  // n_shards * k <= 256 hits per query
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int q = blockIdx.x * kMergePackedWarps + warp;
  if (q >= nq) return;
  PackedHit* mine = stage[warp];
  const int per = k;  // hits of one shard for this query
  for (int i = lane; i < n_shards * per; i += 32) {
    const int g = i / per, j = i % per;
    mine[i] = hits[(static_cast<size_t>(g) * nq + q) * k + j];
  }
  __syncwarp();
  int head = 0;
  for (int i = 0; i < k; ++i) {
    double s = -INFINITY;
    long long r = -1;
    if (lane < n_shards && head < k) {
      const PackedHit h = mine[lane * per + head];
      s = asc ? -h.score : h.score;
      r = h.row;
    }
    // warp arg-max by (score desc, row asc); lanes without a candidate carry r = -1
    double bs = s;
    long long br = r;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const double os = __shfl_xor_sync(0xffffffffu, bs, o);
      const long long orow = __shfl_xor_sync(0xffffffffu, br, o);
      const bool take = orow >= 0 && (br < 0 || os > bs || (os == bs && orow < br));
      bs = take ? os : bs;
      br = take ? orow : br;
    }
    if (r >= 0 && r == br) ++head;  // global rows are unique: exactly one lane advances
    if (lane == 0) {
      const size_t oo = static_cast<size_t>(q) * k + i;
      out_score[oo] = br >= 0 ? static_cast<float>(asc ? -bs : bs) : (asc ? INFINITY : -INFINITY);
      out_idx[oo] = br;
    }
  }
}

// The same merge for any number of shards (<= 64), one thread per query: the fallback of sa_merge_packed_kernel when
// n_shards > 32, k > 32 or n_shards * k > 256, and the merge of sa_merge_shards.  `Hits` loads hit o of the
// [n_shards][nq][k] lists: packed sa_hit records (PackedHits) or separate score and row arrays (SplitHits).
struct PackedHits {
  const PackedHit* __restrict__ hits;
  __device__ __forceinline__ PackedHit at(size_t o) const { return hits[o]; }
};
struct SplitHits {
  const double* __restrict__ score;
  const long long* __restrict__ row;
  __device__ __forceinline__ PackedHit at(size_t o) const { return PackedHit{score[o], row[o]}; }
};
template <typename Hits>
__global__ void sa_merge_serial_kernel(const Hits hits, int n_shards, int nq, int k, float* __restrict__ out_score,
                                       long long* __restrict__ out_idx, int asc) {
  const int q = blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= nq) return;
  int head[64];
  for (int g = 0; g < n_shards; ++g) head[g] = 0;
  for (int i = 0; i < k; ++i) {
    int bg = -1;
    double bs = 0.0;
    long long bi = 0;
    for (int g = 0; g < n_shards; ++g) {
      if (head[g] >= k) continue;
      const PackedHit h = hits.at((static_cast<size_t>(g) * nq + q) * k + head[g]);
      if (h.row < 0) {
        head[g] = k;
        continue;
      }
      const double hs = asc ? -h.score : h.score;
      if (bg < 0 || hs > bs || (hs == bs && h.row < bi)) {
        bg = g;
        bs = hs;
        bi = h.row;
      }
    }
    const size_t oo = static_cast<size_t>(q) * k + i;
    if (bg >= 0) {
      out_score[oo] = static_cast<float>(asc ? -bs : bs);
      out_idx[oo] = bi;
      ++head[bg];
    } else {
      out_score[oo] = asc ? INFINITY : -INFINITY;
      out_idx[oo] = -1;
    }
  }
}

}  // namespace sa
