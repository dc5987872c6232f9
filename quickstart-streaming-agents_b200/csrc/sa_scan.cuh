// The hot path: VECTOR_SEARCH_AGG(<corpus>, DESCRIPTOR(embedding), <query vector>, k)
// (reference call sites: terraform/lab2-vector-search/main.tf:292, LAB3-Walkthrough.md:343-350,
//  LAB4-Walkthrough.md:302-309) as one persistent, warp-specialised sm_90a kernel:
//
//   TMA (SWIZZLE_128B tiles of the bf16 corpus and of the query block)  ->  smem ring
//   wgmma  Q[64 x D] . C[256 x D]^T per consumer warpgroup (two 128-row halves), fp32 accumulators in registers
//   epilogue: accumulators -> smem -> combine with the row's term w[r] -> per-thread (thread == query) sorted register list
//
// The row term w[r] and the epilogue make one kernel serve every similarity of the index (sa_api.h, SA_SIM_*):
//   cosine      v = acc * w, w = 1/|c|     (0 = tombstone)         kEpi = kEpiMul
//   dotProduct  v = acc * w, w = 1         (0 = tombstone)         kEpi = kEpiMul  (the cosine instantiations, unchanged)
//   euclidean   v = acc - w, w = |c|^2 / 2 (negative = tombstone)  kEpi = kEpiSub
// so v is always "larger is better": for euclidean v = <q,c> - |c|^2/2 = (|q|^2 - |q - c|^2) / 2.
// A filtered search (kEpi | kEpiFilt) also masks, per query, the rows whose 64-bit tag fails the query's Filter: their row
// term becomes NaN, exactly like a tombstone's, so an ineligible row never enters a list, raises `drop` or a threshold.
// A deep search (kEpi | kEpiDeep, 28 < k <= 64) keeps the 32-entry lists and changes only the bounds the lanes share
// (kEpiDeep below).
// An int8 index (kEpi | kEpiI8) multiplies int8 rows and queries with s8 wgmma into exact int32 accumulators; a K slice is
// then 128 elements (the same 128 bytes), and the staging buffer receives the accumulators converted to fp32.  From the
// staging buffer on, everything is the bf16 path's.
//
// Nothing but the per-CTA candidate lists (kKL entries per query, plus one "dropped" bound per query) leaves the SM.
//
// Work decomposition.  A "unit" is one CTA (kCG == 1, 128-query blocks) or a cluster of two CTAs (kCG == 2, 256-query
// blocks: each CTA loads half of every corpus slice and multicasts it to both, so the pair reads each corpus tile once).
// Unit u owns query block qb = u % nqb and tile lane tl = u / nqb and walks corpus tiles tl, tl + TL, tl + 2 TL, ...
// (256 rows each: one smem stage holds a K slice of the whole tile, multiplied as two 128-row halves, so the query
// slice crosses L2 once per tile).  All units of one tile lane touch the same corpus tile at about the
// same time (drift control below keeps it so): it crosses HBM once and is served from L2 to the others.
//
// Exactness contract with the merge kernel (sa_aux.cuh).  A thread's list holds the kKL best rows of its tile lane by
// the scan's approximate score a = fp32_accumulate(q.c) * w (or - w), and `drop` is an upper bound on the approximate
// score of every row of the lane that is NOT in the list (evicted, rejected by the own threshold, or rejected by the
// bound shared between lanes).  The merge kernel turns (lists, drops) into either a certificate that the exactly
// re-scored candidates contain the true top-k, or a work item for the exact fallback scan.
#pragma once
#include "sa_aux.cuh"
#include "sm90_ptx.cuh"
#include <cmath>
#include <type_traits>

namespace sa {

constexpr int kBlockM = 128;  // queries per CTA
constexpr int kBlockN = 256;  // corpus rows per tile
constexpr int kHalfN = kWgmmaN;  // corpus rows per MMA: a tile is multiplied as two halves, each into its own accumulators
constexpr int kBlockK = 64;   // bf16 per K slice = 128 B = one swizzle atom
constexpr int kBlockKI8 = 128;  // int8 per K slice: the same 128 B
constexpr int kUmmaK = 16;
constexpr int kScanThreads = 384;  // warpgroup 0: w0 TMA producer; warpgroups 1, 2: 64 queries each (MMA + epilogue)
// Registers per thread after the roles split (setmaxnreg): 128 x 40 + 256 x 232 = 384 x 168, the launch's allocation.
constexpr int kProducerRegs = 40;
constexpr int kConsumerRegs = 232;
constexpr int kChunk = 32;         // columns per list-update chunk
constexpr int kStagingLd = kHalfN + 4;  // floats per query row of the accumulator staging buffer (conflict-free reads)
constexpr int kWin = 16;           // tile lanes whose second-best scores an epilogue thread combines into a bound
constexpr int kWinWarmTiles = 16;  // the window is read on every one of a lane's first tiles, later only after a slow one

// kMode of the scan kernel
constexpr int kModeProd = 0;   // production
constexpr int kModeDots = 1;   // test hook: also dump the raw accumulators of one tile
constexpr int kModeProf = 2;   // profiling: per-role wait / busy cycle counters (ScanParams::prof)

// kEpi of the scan kernel: how the accumulator and the row term combine (see the header comment)
constexpr int kEpiMul = 0;     // v = acc * w; a row is live iff w > 0 (cosine, dotProduct)
constexpr int kEpiSub = 1;     // v = acc - w; a row is live iff w >= 0 (euclidean)
constexpr int kEpiFilt = 2;    // flag: filtered search (ScanParams::row_tags / filters)
constexpr int kEpiDeep = 4;    // flag: deep search (28 < k <= 64 with kKL = 32 entries): bounds valid for the k-th best
constexpr int kEpiI8 = 8;      // flag: int8 rows and queries (s8 wgmma, exact int32 accumulators)
// The int8 K slice occupies the bf16 slice's bytes, so ScanCfg (stage sizes, TMA boxes in bytes, descriptors, staging,
// smem layout) serves both element types unchanged.
static_assert(kBlockKI8 * 1 == kBlockK * 2, "an int8 K slice is one 128-byte swizzle atom, like a bf16 one");

// Deep search.  The list, drop and masking rules are those of every search; only the bounds the lanes share change, since
// a lane's kKL-th best says nothing about a query's k-th best once k > kKL:
//   - a lane does not publish its own kKL-th best into thr_shared (it still reads the slot: the deep pre-pass seeds it
//     with the sample's k-th best, a valid bound for this k);
//   - the window publishes each lane's kDeepWinPos-th best and takes the kDeepWinRank-th largest of the kWin lanes:
//     kDeepWinRank lanes with kDeepWinPos rows scoring >= x each are 70 rows >= x, so x never exceeds the k-th best for
//     any k <= 64 + kDeepMargin (DESIGN.md section 4.1).
constexpr int kShallowMaxK = 28;  // largest k served by the shallow bounds (32-entry lists, 4 spare entries)
constexpr int kDeepMaxK = 64;     // = SA_MAX_K
constexpr int kDeepWinPos = 5;
constexpr int kDeepWinRank = 14;
constexpr int kDeepMargin = kDeepWinPos * kDeepWinRank - kDeepMaxK;
static_assert(kDeepWinRank <= kWin && kDeepMargin >= 6, "the deep window must cover 64 rows plus a margin");

template <int kCG, bool kFilt = false>
struct ScanCfg {
  static constexpr int kStages = 3;
  static constexpr int kBRows = kBlockN / kCG;  // corpus rows of a tile loaded (and multicast) by each CTA
  static constexpr uint32_t kABytes = kBlockM * kBlockK * 2;
  static constexpr uint32_t kBBytes = kBlockN * kBlockK * 2;  // what lands in each CTA per stage
  static constexpr uint32_t kHalfBBytes = kHalfN * kBlockK * 2;  // the second half's rows start this far into B
  static constexpr uint32_t kStageBytes = kABytes + kBBytes;
  static constexpr uint32_t kStagingBytes = kBlockM * kStagingLd * sizeof(float);
  static constexpr uint32_t kIcBytes = 4 * kBlockN * sizeof(float);  // one 256-float scale vector per epilogue warp
  static constexpr uint32_t kBarBytes = 2 * kStages * 8;
  // filtered search: one 256-tag vector per epilogue warp, after the barriers (the unfiltered layout is unchanged)
  static constexpr uint32_t kTagBytes = kFilt ? 4 * kBlockN * sizeof(unsigned long long) : 0;
  // +1024: the dynamic smem base is aligned up to 1024 B by hand (SWIZZLE_128B requirement).
  static constexpr uint32_t kSmemBytes = kStages * kStageBytes + kStagingBytes + kIcBytes + kBarBytes + kTagBytes + 1024;
  static_assert(kSmemBytes <= 227 * 1024, "H100 allows 227 KB of shared memory per block");
  static_assert(!kFilt || kSmemBytes == 228400, "filtered scan: the unfiltered 220 208 B plus 8 KB of tags");
};

// Per-CTA profile record (kModeProf): SM cycles, summed over the kernel.
struct ScanProf {
  long long prod_wait_empty;   // TMA producer blocked on a free smem slot
  long long mma_wait_full;     // first consumer warpgroup blocked on TMA data
  long long mma_wait_tempty;   // first consumer warpgroup blocked on its staging barriers (the other warps' epilogue)
  long long epi_wait_tfull;    // first consumer warpgroup waiting for its last MMAs of a tile to retire
  long long epi_busy;          // first epilogue warp staging and scoring accumulators
  long long epi_slow_chunks;   // 32-column chunks of epilogue warp 0 that took the insertion path
  long long total;             // CTA lifetime
  long long tiles;             // tiles walked
};

struct ScanParams {
  const float* row_term;  // [capacity] w[r] (cosine: 1/|row| over the bf16-rounded row, 0 for an all-zero row or a
                          // tombstone; see kEpi for the others); 16-byte aligned
  long long n_rows;       // committed rows (epoch snapshot); rows >= n_rows are masked
  int nq;                 // queries covered by tmap_q
  int num_kb;             // K slices: D / 64 (int8: D / 128)
  int num_tiles;          // ceil(n_rows / 256)
  int nqb;                // query blocks of 128*kCG rows
  int tl_count;           // tile lanes (TL)
  float* part_score;      // [gridDim.x][128][kKL]
  int* part_idx;          // [gridDim.x][128][kKL]
  float* part_drop;       // [gridDim.x][128]  upper bound on the approximate score of the lane's rows not in the list
  int corpus_evict_first; // 1: corpus tiles are read by a single query block -> stream them through L2
  int tile_stride;        // 1: walk every tile; S > 1: the sampling pre-pass walks tiles 0, S, 2S, ... only
  int wait_hint_ns;       // suspend-time hint of the consumers' mbarrier waits (0 = plain polling)
  int* lane_progress;     // [tl_count][nqb] tiles whose loads each unit has issued (zero at launch), or nullptr
  int unit_map;           // 0: unit = tl*nqb + qb (lane-mates adjacent), 1: unit = qb*TL + tl (lane-mates TL apart)
  int max_drift;          // lead (in tiles) over the slowest lane-mate that is not paced
  int pace_gain;          // SM cycles of delay per K-slice issue per tile of lead beyond max_drift (0 = free-running)
  int pace_max;           // cap of that delay
  unsigned* thr_shared;   // [nqb*128*kCG] per-query lower bound on the kKL-th best score (deep search: on the k-th best,
                          // seeded by the pre-pass only), order-preserving keys (zero at launch), or nullptr: lanes then
                          // learn their thresholds alone
  unsigned* lane2;        // [tl_count][nqb*128*kCG] each lane's SECOND-best score per query (deep search: its
                          // kDeepWinPos-th best; keys, zero at launch), or
                          // nullptr.  kKL/2 lanes with two rows >= x each are kKL rows >= x: a much tighter bound than
                          // any single lane's kKL-th best while the lists are young (window_bound below)
  long long* dbg_times;   // optional [gridDim.x][2]: globaltimer at CTA start / end (ns), for drift studies
  float* dbg_dots;        // kModeDots only: raw accumulators of (unit 0 .. nqb-1, tile dbg_tile) [nqb*128*kCG][256]
  int dbg_tile;
  ScanProf* prof;         // kModeProf only: [gridDim.x]
  const unsigned long long* row_tags;  // kEpiFilt only: [capacity] the rows' tags, 16-byte aligned (rows < n_rows read)
  const Filter* filters;               // kEpiFilt only: [nq] this launch's queries' filters
};

// The largest float strictly less than x (x finite): `s > float_below(x)` <=> `s >= x`.
__host__ __device__ __forceinline__ float float_below(float x) {
  const int b = static_cast<int>(f32_bits(x));
  if (x > 0.f) return bits_f32(static_cast<unsigned>(b - 1));
  if (x < 0.f) return bits_f32(static_cast<unsigned>(b + 1));
  return bits_f32(0x80000001u);  // below +-0: the smallest negative denormal
}

// max that ignores a NaN operand (device: FMNMX; host: the same rule spelled out for the CPU unit tests)
__host__ __device__ __forceinline__ float max_nn(float a, float b) {
#ifdef __CUDA_ARCH__
  return fmaxf(a, b);
#else
  if (a != a) return b;
  if (b != b) return a;
  if (a == b) return (f32_bits(a) & 0x80000000u) ? b : a;  // max(+0, -0) = +0, as FMNMX
  return a > b ? a : b;
#endif
}

// Sorted (descending score, ascending row on ties) insertion into a register-resident list.
// Precondition: s > sc[kKL-1].  Rows reach a thread in ascending order, so a strict compare keeps the
// lower row index ahead of an equal score.
template <int kKL>
__host__ __device__ __forceinline__ void list_insert(float (&sc)[kKL], int (&id)[kKL], float s, int row) {
#ifdef __CUDA_ARCH__
#pragma unroll
#endif
  for (int i = kKL - 1; i > 0; --i) {
    const bool shift = s > sc[i - 1];
    const bool here = s > sc[i];
    const float ns = shift ? sc[i - 1] : (here ? s : sc[i]);
    const int ni = shift ? id[i - 1] : (here ? row : id[i]);
    sc[i] = ns;
    id[i] = ni;
  }
  if (s > sc[0]) {
    sc[0] = s;
    id[0] = row;
  }
}

// The window bound.  Every tile lane publishes, per query, the SECOND best score it holds.  If kKL/2 different lanes each
// hold two rows scoring >= x, kKL rows score >= x (lanes own disjoint rows), so no row scoring < x is in the query's
// global top-kKL: x = the (kKL/2)-th largest of the lanes' second bests is a valid shared bound.  After t tiles per
// lane it sits near the top 1.7/(256 t) of the scores, the best single lane's kKL-th best near 9/(256 t): about five
// times fewer values pass it, which is what the first tiles of a short scan spend their time on.  16 keys, bitonic
// network (80 compare-exchanges, branch-free; key 0 = nothing published sorts last, so an early window yields 0 = no bound).
__host__ __device__ __forceinline__ void sort16_desc(unsigned (&x)[kWin]) {
  static_assert(kWin == 16, "the network below is the 16-input bitonic sorter");
#ifdef __CUDA_ARCH__
#pragma unroll
#endif
  for (int k = 2; k <= 16; k <<= 1) {
#ifdef __CUDA_ARCH__
#pragma unroll
#endif
    for (int j = k >> 1; j > 0; j >>= 1) {
#ifdef __CUDA_ARCH__
#pragma unroll
#endif
      for (int i = 0; i < 16; ++i) {
        const int l = i ^ j;
        if (l > i) {
          const unsigned a = x[i], b = x[l];
          const unsigned hi = a > b ? a : b, lo = a > b ? b : a;
          const bool desc = (i & k) == 0;
          x[i] = desc ? hi : lo;
          x[l] = desc ? lo : hi;
        }
      }
    }
  }
}
// Deep search (kDeep): x[i] is lane i's kDeepWinPos-th best.  If kDeepWinRank different lanes each hold kDeepWinPos rows
// scoring >= x, 70 rows score >= x: the kDeepWinRank-th largest bounds the k-th best for every k <= 70 (key 0 = no bound).
template <int kKL, bool kDeep = false>
__host__ __device__ __forceinline__ unsigned window_bound(unsigned (&x)[kWin]) {
  static_assert(kKL / 2 <= kWin, "the window must hold kKL/2 lanes");
  sort16_desc(x);
  return x[(kDeep ? kDeepWinRank : kKL / 2) - 1];
}

// One query's candidate list as an epilogue thread holds it: all indices are compile-time, so it lives in registers.
template <int kKL>
struct TopList {
  float sc[kKL];
  int id[kKL];
  float thr;        // current insertion threshold = max(own kKL-th best, thr_floor)
  float thr_floor;  // largest float strictly below the bound shared by the other tile lanes
  float published;  // last own kKL-th best written to the shared bound
  float drop;       // max approximate score of any row this thread saw and does not hold (NaN-free; -inf = none)
  unsigned nxt_key; // shared bound fetched at the end of the previous accumulator (0 = nothing published yet)
  unsigned* slot;   // this query's shared bound (or nullptr)
  __host__ __device__ __forceinline__ void init(unsigned* shared_slot) {
#ifdef __CUDA_ARCH__
#pragma unroll
#endif
    for (int i = 0; i < kKL; ++i) {
      sc[i] = -INFINITY;
      id[i] = -1;
    }
    thr = thr_floor = published = drop = -INFINITY;
    nxt_key = 0u;
    slot = shared_slot;
  }
  // a bound published by another tile lane becomes visible
  __host__ __device__ __forceinline__ void apply_shared(unsigned key) {
    if (key != 0u) {
      thr_floor = max_nn(thr_floor, float_below(key_to_float(key)));  // bounds only ever tighten
      thr = max_nn(thr, thr_floor);
    }
  }
};

// One 32-column chunk: scale, reduce to the chunk maximum with full instruction-level parallelism, and only when that
// beats the threshold (probability ~ 32 kKL / n after n rows) take the insertion path.  Returns true if it ran.
//
// Insertion path: extract-max rounds over the whole chunk -- each round takes the thread's largest remaining value (the
// lowest row among equals), inserts it, masks it and re-reduces -- until nothing beats the threshold.  A warp executes
// as many rounds as its busiest lane needs (usually one or two), however the qualifying values are spread over the 32
// rows; walking the rows group by group instead costs a round per group that ANY lane has a hit in, which during the
// warm-up of a short scan (few tiles per lane) dominates the epilogue's time.
template <int kKL, int kEpi = kEpiMul>
__host__ __device__ __forceinline__ bool chunk_process(TopList<kKL>& L, float (&v)[kChunk], const float (&w)[kChunk],
                                                       int row_base) {
  auto reduce = [&]() {
    float g[8];
#ifdef __CUDA_ARCH__
#pragma unroll
#endif
    for (int i = 0; i < 8; ++i)
      g[i] = max_nn(max_nn(v[4 * i + 0], v[4 * i + 1]), max_nn(v[4 * i + 2], v[4 * i + 3]));
    return max_nn(max_nn(max_nn(g[0], g[1]), max_nn(g[2], g[3])), max_nn(max_nn(g[4], g[5]), max_nn(g[6], g[7])));
  };
#ifdef __CUDA_ARCH__
#pragma unroll
#endif
  for (int i = 0; i < kChunk; ++i) {
    if constexpr (kEpi == kEpiSub)
      v[i] -= w[i];
    else
      v[i] *= w[i];
  }
  float m = reduce();
  if (!(m > L.thr)) {
    L.drop = max_nn(L.drop, m);
    return false;
  }
  do {
    int pos = kChunk - 1;
#ifdef __CUDA_ARCH__
#pragma unroll
#endif
    for (int j = kChunk - 2; j >= 0; --j) pos = (v[j] == m) ? j : pos;  // lowest row among equals first
    float sj = m;
    if (m == 0.f) {  // keep the element's own sign of zero (max(+0, -0) is +0)
#ifdef __CUDA_ARCH__
#pragma unroll
#endif
      for (int j = 0; j < kChunk; ++j) sj = (j == pos) ? v[j] : sj;
    }
#ifdef __CUDA_ARCH__
#pragma unroll
#endif
    for (int j = 0; j < kChunk; ++j) v[j] = (j == pos) ? -INFINITY : v[j];
    L.drop = max_nn(L.drop, L.sc[kKL - 1]);  // the evicted tail (-inf while the list fills)
    list_insert<kKL>(L.sc, L.id, sj, row_base + pos);
    L.thr = max_nn(L.sc[kKL - 1], L.thr_floor);
    m = reduce();
  } while (m > L.thr);
  L.drop = max_nn(L.drop, m);  // whatever is left of the chunk was rejected (NaN = masked rows: ignored)
  return true;
}

#ifdef __CUDACC__
// Epilogue of one half tile: 128 columns of this thread's query row in the staging buffer -> scaled scores -> list.
// `ic` is this warp's private 256-float scale vector of the tile in shared memory (broadcast reads).
// Filtered (kEpi & kEpiFilt): `tg` is the warp's tag vector of the half, and a row failing the thread's filter `*fp`
// gets the row term NaN (acc * NaN and acc - NaN are NaN: masked like a tombstone).  The filter is re-read (L1) and
// reduced to a 32-bit pass mask per chunk before the chunk's values are loaded, so it holds no registers in between.
template <int kKL, int kMode, int kEpi>
__device__ __forceinline__ int epilogue_half(TopList<kKL>& L, const float* srow, const float* ic, int row0,
                                             float* dbg_row, const unsigned long long* tg = nullptr,
                                             const Filter* fp = nullptr) {
  int slow = 0;
  float v[kChunk], w[kChunk];
#pragma unroll 1
  for (int c = 0; c < kHalfN / kChunk; ++c) {
    unsigned pass = 0u;
    if constexpr ((kEpi & kEpiFilt) != 0) {
      const Filter F = *fp;
#pragma unroll
      for (int j = 0; j < kChunk; ++j) pass |= filter_pass(tg[c * kChunk + j], F) ? (1u << j) : 0u;
    }
    const float4* s4 = reinterpret_cast<const float4*>(srow + c * kChunk);
    const float4* w4 = reinterpret_cast<const float4*>(ic + c * kChunk);
#pragma unroll
    for (int i = 0; i < kChunk / 4; ++i) {
      const float4 x = s4[i], y = w4[i];
      v[4 * i + 0] = x.x;
      v[4 * i + 1] = x.y;
      v[4 * i + 2] = x.z;
      v[4 * i + 3] = x.w;
      w[4 * i + 0] = y.x;
      w[4 * i + 1] = y.y;
      w[4 * i + 2] = y.z;
      w[4 * i + 3] = y.w;
    }
    if constexpr ((kEpi & kEpiFilt) != 0) {
      const float qnan = __int_as_float(0x7fc00000);
#pragma unroll
      for (int j = 0; j < kChunk; ++j) w[j] = ((pass >> j) & 1u) ? w[j] : qnan;
    }
    if constexpr (kMode == kModeDots) {
      if (dbg_row != nullptr) {
#pragma unroll
        for (int j = 0; j < kChunk; ++j) dbg_row[c * kChunk + j] = v[j];
      }
    }
    slow += chunk_process<kKL, kEpi & 1>(L, v, w, row0 + c * kChunk) ? 1 : 0;
    __syncwarp();  // reconverge after the divergent insertion path
  }
  return slow;
}

template <int kCG, int kKL, int kMode, int kEpi = kEpiMul>
__global__ void __launch_bounds__(kScanThreads, 1)
sa_scan_kernel(const __grid_constant__ CUtensorMap tmap_q, const __grid_constant__ CUtensorMap tmap_c,
               const ScanParams p) {
  constexpr bool kFilt = (kEpi & kEpiFilt) != 0;
  constexpr bool kDeep = (kEpi & kEpiDeep) != 0;
  constexpr bool kI8 = (kEpi & kEpiI8) != 0;
  constexpr int kSliceK = kI8 ? kBlockKI8 : kBlockK;  // elements per K slice (the TMA box's x extent)
  using Acc = typename std::conditional<kI8, int, float>::type;
  static_assert(!kDeep || (kKL == 32 && kMode == kModeProd), "deep search: 32-entry lists, production build only");
  using Cfg = ScanCfg<kCG, kFilt>;
  static_assert(!(kDeep && kFilt) || Cfg::kSmemBytes == 228400, "the filtered deep scan has its twin's smem layout");
  constexpr int kStages = Cfg::kStages;
  constexpr int kRowsPerQb = kBlockM * kCG;
  constexpr bool kProf = (kMode == kModeProf);

  extern __shared__ uint8_t smem_raw[];
  const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  uint8_t* smem_gen = smem_raw + (smem_base - smem_u32(smem_raw));

  float* staging = reinterpret_cast<float*>(smem_gen + kStages * Cfg::kStageBytes);  // [128 queries][kStagingLd]
  float* icbuf = reinterpret_cast<float*>(smem_gen + kStages * Cfg::kStageBytes + Cfg::kStagingBytes);  // [4][256]
  const uint32_t bar_base = smem_base + kStages * Cfg::kStageBytes + Cfg::kStagingBytes + Cfg::kIcBytes;
  auto full_bar = [&](int s) { return bar_base + 8u * s; };
  auto empty_bar = [&](int s) { return bar_base + 8u * (kStages + s); };
  auto a_smem = [&](int s) { return smem_base + s * Cfg::kStageBytes; };
  auto b_smem = [&](int s) { return smem_base + s * Cfg::kStageBytes + Cfg::kABytes; };
  const uint32_t tag_base = bar_base + Cfg::kBarBytes;  // [4][256] tags (kFilt only)

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const uint32_t rank = (kCG == 2) ? cluster_ctarank() : 0u;
  const int TL = p.tl_count;
  const int nqb = p.nqb;  // units per tile lane
  // This unit's query block, tile lane and the tiles this launch visits (all lanes together).  Each role computes them
  // after its setmaxnreg: ptxas keeps a value that is live across the register reallocation in local memory.
  struct Walk {
    int qb, tl, tiles;
  };
  auto walk_of = [&]() {
    const int unit = blockIdx.x / kCG;
    Walk w;
    w.qb = p.unit_map == 0 ? unit % nqb : unit / TL;
    w.tl = p.unit_map == 0 ? unit / nqb : unit % TL;
    w.tiles = (p.num_tiles + p.tile_stride - 1) / p.tile_stride;
    return w;
  };

  // ------------------------------------------------------------------ one-time setup
  long long t_start = 0;
  if constexpr (kProf) t_start = clock64();
  if (p.dbg_times != nullptr && threadIdx.x == 0) p.dbg_times[2 * blockIdx.x] = globaltimer_ns();
  if (warp == 0 && lane == 0) {
    tma_prefetch_desc(&tmap_q);
    tma_prefetch_desc(&tmap_c);
  }
  if (warp == 1 && lane == 0) {
    for (int s = 0; s < kStages; ++s) {
      mbar_init(full_bar(s), 1);         // this CTA producer's arrive.expect_tx; TMA bytes complete it
      mbar_init(empty_bar(s), 2 * kCG);  // one arrive per consumer warpgroup of every CTA the slot is multicast to
    }
    fence_mbar_init();
  }
  __syncthreads();
  if constexpr (kCG == 2) cluster_sync_all();  // the peer's barriers are initialised before any multicast or remote arrive

  // ------------------------------------------------------------------ roles
  if (warp < 4) {
    setmaxnreg_dec<kProducerRegs>();  // the whole warpgroup: only w0's lane 0 has work
    if (warp == 0 && lane == 0) {
      // ===== TMA producer =====
      const Walk w = walk_of();
      const int qb = w.qb, tl = w.tl, walk_tiles = w.tiles;
      const uint64_t c_hint = p.corpus_evict_first ? kEvictFirst : kEvictNormal;
      int stage = 0;
      uint32_t phase = 0;
      long long waited = 0;
      // Drift control between the units of a tile lane.  Units that share a corpus tile run identical work but at
      // slightly different speeds, so over thousands of tiles they drift tens of tiles apart; once the spread exceeds
      // what L2 holds, every unit re-reads its tiles from HBM.  A hard barrier costs a pipeline drain per tile, so the
      // leader producers *pace* themselves instead: each publishes how many tiles it has issued, reads its
      // lane-mates' counters once per tile, and a unit that leads the slowest mate by more than `max_drift` tiles
      // delays every K-slice issue by pace_gain cycles per extra tile of lead (capped).  The kernel's duration is
      // set by its slowest unit anyway, so slowing the fast ones is free; it is only a hint (no waiting on
      // anyone), hence no co-residency assumption and no deadlock.
      const bool lockstep = p.lane_progress != nullptr && p.pace_gain > 0 && nqb > 1 && rank == 0;
      int pace = 0;
      int tile_no = 0;
      const int q_row = qb * kRowsPerQb + static_cast<int>(rank) * kBlockM;
      for (int ti = tl; ti < walk_tiles; ti += TL, ++tile_no) {
        const int t = ti * p.tile_stride;
        if (lockstep) {
          const int* pr = p.lane_progress + tl * nqb;
          int slowest = tile_no;
          for (int j = 0; j < nqb; ++j) slowest = min(slowest, ld_relaxed_gpu(pr + j));
          pace = min(max(tile_no - slowest - p.max_drift, 0) * p.pace_gain, p.pace_max);
        }
        // one stage per K slice: the query slice and the whole tile's corpus slice (each CTA of a pair loads its
        // kBRows rows and multicasts them to both)
        const int c_row = t * kBlockN + static_cast<int>(rank) * Cfg::kBRows;
        for (int kb = 0; kb < p.num_kb; ++kb) {
          if constexpr (kProf) {
            const long long c0 = clock64();
            mbar_wait(empty_bar(stage), phase ^ 1u);
            waited += clock64() - c0;
          } else {
            mbar_wait(empty_bar(stage), phase ^ 1u);  // consumers of every CTA sharing the slot have released it
          }
          if (pace > 0) {
            const long long c0 = clock64();
            while (clock64() - c0 < pace) {
            }
          }
          mbar_expect_tx(full_bar(stage), Cfg::kStageBytes);
          tma_load_2d(a_smem(stage), &tmap_q, full_bar(stage), kb * kSliceK, q_row, kEvictLast);
          const uint32_t b_dst = b_smem(stage) + rank * (Cfg::kBRows * kBlockK * 2);
          if constexpr (kCG == 1)
            tma_load_2d(b_dst, &tmap_c, full_bar(stage), kb * kSliceK, c_row, c_hint);
          else
            tma_load_2d_multicast(b_dst, &tmap_c, full_bar(stage), kb * kSliceK, c_row, 0x3, c_hint);
          if (++stage == kStages) {
            stage = 0;
            phase ^= 1u;
          }
        }
        if (lockstep) st_relaxed_gpu(p.lane_progress + tl * nqb + qb, tile_no + 1);
      }
      if constexpr (kProf) {
        p.prof[blockIdx.x].prod_wait_empty = waited;
        p.prof[blockIdx.x].tiles = tile_no;
      }
    }
  } else {
    // ===== consumers: warpgroup g (1 or 2) multiplies queries [64 (g-1), 64 g) of the block with each tile, one
    // accumulator set per 128-row half, stages each half's accumulators in smem in turn, and its first two warps
    // (thread == query) feed them to the candidate lists.  The two warpgroups only meet at the smem ring's barriers. =====
    setmaxnreg_inc<kConsumerRegs>();  // both accumulator sets stay live through the first half's epilogue
    const Walk w = walk_of();
    const int qb = w.qb, tl = w.tl, walk_tiles = w.tiles;
    const int g = warp / 4 - 1;
    const int wt = threadIdx.x & 127;          // thread within the warpgroup
    const bool epi = (warp & 3) < 2;           // epilogue warp: its 32 lanes own 32 of the warpgroup's 64 queries
    const int ew = 2 * g + (warp & 3);         // epilogue warp index within the CTA (valid when epi)
    const int et = 64 * g + wt;                // query row within the CTA's block (valid when epi)
    const bool signaller = wt == 0;            // releases smem slots and keeps the profile counters
    const uint32_t named_bar = 1 + g;
    float* ic = icbuf + ew * kBlockN;
    float* stg = staging + 64 * g * kStagingLd;
    // Threshold sharing.  A thread's list only ever sees its own tile lane, so alone it needs ~kKL*ln(n) insertions
    // to warm up, and a warp pays for every lane's insertions.  But if ANY lane already holds kKL rows scoring >= x
    // for this query, no row scoring < x can be in the query's global top-kKL.  So each epilogue thread publishes its
    // kKL-th best (atomicMax on an order-preserving key) and reads the shared bound once per tile: every lane gets the
    // threshold of the whole machine's progress, and the warm-up tail disappears (a deep search publishes nothing here:
    // its k-th best may lie past any lane's kKL-th best).  The shared bound admits ties (>=),
    // the thread's own bound stays strict (>), so tie-breaking by row is unchanged.
    const int query = qb * kRowsPerQb + static_cast<int>(rank) * kBlockM + et;
    const bool own_query = epi && query < p.nq;
    TopList<kKL> L;
    L.init((p.thr_shared != nullptr && own_query) ? p.thr_shared + query : nullptr);

    // Row terms of tile t: lane l fetches rows [8l, 8l+8) (two 16-byte loads), masks rows past the committed prefix
    // and rows that are not live (all-zero rows under cosine, tombstones) with NaN (NaN never compares greater than a
    // threshold, so they cannot enter a list and are ignored by every max), and the warp shares them through its
    // private smem vector.  Past the prefix the term reads as kPast, which every epilogue masks.
    constexpr float kPast = ((kEpi & 1) == kEpiSub) ? -1.f : 0.f;
    float4 nx0 = make_float4(0.f, 0.f, 0.f, 0.f), nx1 = nx0;
    auto fetch_ic = [&](int t) {
      const long long r0 = static_cast<long long>(t) * kBlockN + 8 * lane;
      const float4* src = reinterpret_cast<const float4*>(p.row_term + r0);
      if (r0 + 8 <= p.n_rows) {
        nx0 = __ldg(src);
        nx1 = __ldg(src + 1);
      } else {
        float x[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) x[j] = (r0 + j < p.n_rows) ? __ldg(p.row_term + r0 + j) : kPast;
        nx0 = make_float4(x[0], x[1], x[2], x[3]);
        nx1 = make_float4(x[4], x[5], x[6], x[7]);
      }
    };
    if (epi && tl < walk_tiles) fetch_ic(tl * p.tile_stride);
    // Tags of tile t (kFilt): lane l copies rows [8l, 8l+8) into the warp's private vector with cp.async, issued once
    // the warp's previous epilogue is done with the vector and waited for at the start of the next epilogue, so the
    // copy holds no registers across the MMAs.  Tags at or past n_rows are not read (zero-filled; those rows are masked).
    auto fetch_tags = [&](int t) {
      const long long r0 = static_cast<long long>(t) * kBlockN + 8 * lane;
      const uint32_t dst = tag_base + static_cast<uint32_t>((ew * kBlockN + 8 * lane) * sizeof(unsigned long long));
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const long long left = p.n_rows - (r0 + 2 * j);
        const uint32_t bytes = left >= 2 ? 16u : (left == 1 ? 8u : 0u);
        cp_async_16(dst + 16u * j, p.row_tags + (bytes != 0u ? r0 + 2 * j : 0), bytes);
      }
    };
    if constexpr (kFilt) {
      if (epi && tl < walk_tiles) fetch_tags(tl * p.tile_stride);
    }

    // Window bound (see window_bound): this thread's slot in the lanes' second-best table, and the kWin lanes it reads.
    const bool win_on = p.lane2 != nullptr && TL >= kWin && own_query;
    const size_t win_stride = static_cast<size_t>(p.nqb) * kRowsPerQb;
    unsigned* const win_q = win_on ? p.lane2 + query : nullptr;
    float pub2 = -INFINITY;   // last second-best published
    unsigned nx2[kWin] = {};  // the window as read at the end of the previous tile
    bool have2 = false;

    const uint64_t a_desc0 = make_kmajor_sw128_desc(a_smem(0) + g * (64 * kBlockK * 2));
    const uint64_t b_desc0 = make_kmajor_sw128_desc(b_smem(0));
    constexpr uint64_t kStageDesc = Cfg::kStageBytes >> 4;  // one stage further in the descriptors' address field
    constexpr uint64_t kHalfBDesc = Cfg::kHalfBBytes >> 4;  // the tile's second half in B
    int stage = 0;
    uint32_t phase = 0;
    long long w_full = 0, w_stage = 0, w_mma = 0, busy = 0, slow_chunks = 0;
    for (int ti = tl; ti < walk_tiles; ti += TL) {
      const int t = ti * p.tile_stride;
      int slow = 0;
      if (epi) {
        if (have2) {
          const unsigned kb = window_bound<kKL, kDeep>(nx2);
          L.nxt_key = kb > L.nxt_key ? kb : L.nxt_key;
          have2 = false;
        }
        L.apply_shared(L.nxt_key);
        const float qnan = __int_as_float(0x7fc00000);
        auto sc = [&](float x) {
          if constexpr ((kEpi & 1) == kEpiSub)
            return x >= 0.f ? x : qnan;
          else
            return x > 0.f ? x : qnan;
        };
        float4* dst = reinterpret_cast<float4*>(ic + 8 * lane);
        dst[0] = make_float4(sc(nx0.x), sc(nx0.y), sc(nx0.z), sc(nx0.w));
        dst[1] = make_float4(sc(nx1.x), sc(nx1.y), sc(nx1.z), sc(nx1.w));
        __syncwarp();  // ic[] visible to the whole warp
      }
      // The window is consumed.  Cleared on every path, it holds no value across the MMAs: the compiler cannot tell
      // that `have2` is false until the next fetch, and would otherwise keep kWin registers live through the tile.
#pragma unroll
      for (int i = 0; i < kWin; ++i) nx2[i] = 0u;
      float* dbg_row = nullptr;
      if constexpr (kMode == kModeDots) {
        if (own_query && p.dbg_dots != nullptr && t == p.dbg_tile) dbg_row = p.dbg_dots + static_cast<size_t>(query) * kBlockN;
      }
      // ---- MMA: acc0 = Q[64 x D] . C[rows 0..127 of the tile]^T, acc1 the same for rows 128..255, K slice by K slice,
      // both from the same A slice; a slot is released once the MMAs reading it have retired (wait_group 1 after the
      // next slice's issue keeps one slice in flight)
      Acc acc0[64], acc1[64];  // dead between tiles: the first MMA of a tile overwrites them
      int prev_stage = -1;
      for (int kb = 0; kb < p.num_kb; ++kb) {
        if constexpr (kProf) {
          const long long c0 = clock64();
          mbar_wait(full_bar(stage), phase, static_cast<uint32_t>(p.wait_hint_ns));
          w_full += clock64() - c0;
        } else {
          mbar_wait(full_bar(stage), phase, static_cast<uint32_t>(p.wait_hint_ns));
        }
        wgmma_fence();
        wgmma_fence_operands(acc0);
        wgmma_fence_operands(acc1);
#pragma unroll
        for (int k = 0; k < kBlockK / kUmmaK; ++k) {
          // +32 B along K inside the 128-B swizzle atom (16 bf16 or 32 int8) = +2 in the (addr >> 4) field
          const uint64_t a_desc = a_desc0 + stage * kStageDesc + 2u * k;
          const uint64_t b_desc = b_desc0 + stage * kStageDesc + 2u * k;
          if constexpr (kI8) {
            wgmma_m64n128k32_s8(acc0, a_desc, b_desc, (kb | k) != 0 ? 1u : 0u);
            wgmma_m64n128k32_s8(acc1, a_desc, b_desc + kHalfBDesc, (kb | k) != 0 ? 1u : 0u);
          } else {
            wgmma_m64n128k16_bf16(acc0, a_desc, b_desc, (kb | k) != 0 ? 1u : 0u);
            wgmma_m64n128k16_bf16(acc1, a_desc, b_desc + kHalfBDesc, (kb | k) != 0 ? 1u : 0u);
          }
        }
        wgmma_commit();
        wgmma_fence_operands(acc0);
        wgmma_fence_operands(acc1);
        if (prev_stage >= 0) {
          wgmma_wait<1>();
          if (signaller) {
            mbar_arrive(empty_bar(prev_stage));
            if constexpr (kCG == 2) mbar_arrive_cluster(empty_bar(prev_stage), rank ^ 1u);
          }
        }
        prev_stage = stage;
        if (++stage == kStages) {
          stage = 0;
          phase ^= 1u;
        }
      }
      long long c0 = 0;
      if constexpr (kProf) c0 = clock64();
      wgmma_wait<0>();
      wgmma_fence_operands(acc0);
      wgmma_fence_operands(acc1);
      if (signaller) {
        mbar_arrive(empty_bar(prev_stage));
        if constexpr (kCG == 2) mbar_arrive_cluster(empty_bar(prev_stage), rank ^ 1u);
      }
      if constexpr (kProf) w_mma += clock64() - c0;
      // prefetch the next tile's row terms: issued after the MMAs, so that they hold no registers across them
      if (epi && ti + TL < walk_tiles) fetch_ic((ti + TL) * p.tile_stride);
      // ---- one half at a time through the staging buffer, rows in ascending order
      // int8: the exact int32 accumulator rounded once to fp32 (the scan's only accumulation error)
      auto to_f32 = [](Acc x) {
        if constexpr (kI8)
          return __int2float_rn(x);
        else
          return x;
      };
      auto stage_and_score = [&](const Acc (&acc)[64], int h) {
        long long c1 = 0;
        if constexpr (kProf) c1 = clock64();
        named_bar_sync(named_bar, 128);  // the previous half's readers are done with the buffer
#pragma unroll
        for (int j = 0; j < 16; ++j) {
          const int r = 16 * (wt >> 5) + ((wt & 31) >> 2);
          const int col = 8 * j + 2 * (wt & 3);
          *reinterpret_cast<float2*>(stg + r * kStagingLd + col) =
              make_float2(to_f32(acc[4 * j + 0]), to_f32(acc[4 * j + 1]));
          *reinterpret_cast<float2*>(stg + (r + 8) * kStagingLd + col) =
              make_float2(to_f32(acc[4 * j + 2]), to_f32(acc[4 * j + 3]));
        }
        named_bar_sync(named_bar, 128);
        long long c2 = 0;
        if constexpr (kProf) c2 = clock64();
        if constexpr (kFilt) {
          if (epi && h == 0) {
            cp_async_wait_all();
            __syncwarp();  // every lane's tags of this tile are in the warp's vector
          }
        }
        if constexpr (kFilt) {
          // this warp's tag vector, formed here rather than held across the MMAs
          const unsigned long long* tg =
              reinterpret_cast<const unsigned long long*>(smem_gen + (tag_base - smem_base)) + ew * kBlockN;
          if (epi)
            slow += epilogue_half<kKL, kMode, kEpi>(L, stg + wt * kStagingLd, ic + h * kHalfN, t * kBlockN + h * kHalfN,
                                                    dbg_row != nullptr ? dbg_row + h * kHalfN : nullptr, tg + h * kHalfN,
                                                    p.filters + (own_query ? query : 0));
        } else if (epi) {
          slow += epilogue_half<kKL, kMode, kEpi>(L, stg + wt * kStagingLd, ic + h * kHalfN, t * kBlockN + h * kHalfN,
                                                  dbg_row != nullptr ? dbg_row + h * kHalfN : nullptr);
        }
        if constexpr (kProf) {
          w_stage += c2 - c1;
          busy += clock64() - c2;
        }
      };
      stage_and_score(acc0, 0);
      stage_and_score(acc1, 1);
      if constexpr (kFilt) {
        if (epi && ti + TL < walk_tiles) {
          __syncwarp();  // every lane is done reading this tile's tags
          fetch_tags((ti + TL) * p.tile_stride);
        }
      }
      if constexpr (kProf) slow_chunks += slow;
      if (epi) {
        if (L.slot != nullptr) {
          // list full and its tail improved: tell the other lanes (a deep search's k-th best may lie past the tail)
          if constexpr (!kDeep) {
            if (L.sc[kKL - 1] > L.published) {
              L.published = L.sc[kKL - 1];
              atomicMax(L.slot, float_to_key(L.published));
            }
          }
          L.nxt_key = ld_relaxed_gpu_u32(L.slot);  // consumed at the start of the next tile: latency hidden
        }
        // publish this lane's second best (deep: kDeepWinPos-th best) and, while the lists are young (or whenever a
        // warp just paid for insertions), fetch the window for the next tile's bound
        if (p.lane2 != nullptr && TL >= kWin) {
          const bool fetch = (ti - tl) / TL < kWinWarmTiles || __any_sync(0xffffffffu, slow > 0);
          if (win_on) {
            constexpr int kPub = kDeep ? kDeepWinPos - 1 : 1;
            if (L.sc[kPub] > pub2) {
              pub2 = L.sc[kPub];
              st_relaxed_gpu_u32(win_q + static_cast<size_t>(tl) * win_stride, float_to_key(pub2));
            }
            if (fetch && ti + TL < walk_tiles) {
              // the stride goes through an opaque move so that the kWin addresses are formed here, at each fetch:
              // hoisted out of the tile loop they would hold 2 kWin registers across the MMAs, and spill
              size_t stride = win_stride;
              asm volatile("" : "+l"(stride));
#pragma unroll
              for (int i = 0; i < kWin; ++i) {
                int ln = tl + i;
                ln -= (ln >= TL) ? TL : 0;
                nx2[i] = ld_relaxed_gpu_u32(win_q + static_cast<size_t>(ln) * stride);
              }
              have2 = true;
            }
          }
        }
      }
    }

    // The only global writes of the scan: this CTA's candidate list and drop bound for each of its queries.
    if (own_query) {
      const size_t o = (static_cast<size_t>(blockIdx.x) * kBlockM + et) * kKL;
      float4* ps = reinterpret_cast<float4*>(p.part_score + o);
      int4* pi = reinterpret_cast<int4*>(p.part_idx + o);
#pragma unroll
      for (int i = 0; i < kKL / 4; ++i) {
        ps[i] = make_float4(L.sc[4 * i], L.sc[4 * i + 1], L.sc[4 * i + 2], L.sc[4 * i + 3]);
        pi[i] = make_int4(L.id[4 * i], L.id[4 * i + 1], L.id[4 * i + 2], L.id[4 * i + 3]);
      }
      p.part_drop[static_cast<size_t>(blockIdx.x) * kBlockM + et] = L.drop;
    }
    if constexpr (kProf) {
      if (g == 0 && signaller) {
        p.prof[blockIdx.x].mma_wait_full = w_full;
        p.prof[blockIdx.x].mma_wait_tempty = w_stage;
        p.prof[blockIdx.x].epi_wait_tfull = w_mma;
        p.prof[blockIdx.x].epi_busy = busy;
        p.prof[blockIdx.x].epi_slow_chunks = slow_chunks;
      }
    }
  }

  // ------------------------------------------------------------------ teardown
  __syncthreads();
  if (p.dbg_times != nullptr && threadIdx.x == 0) p.dbg_times[2 * blockIdx.x + 1] = globaltimer_ns();
  if constexpr (kProf) {
    if (threadIdx.x == 0) p.prof[blockIdx.x].total = clock64() - t_start;
  }
  if constexpr (kCG == 2) cluster_sync_all();  // the peer may still be multicasting into our smem / arriving on our barriers
}
#endif  // __CUDACC__

}  // namespace sa
