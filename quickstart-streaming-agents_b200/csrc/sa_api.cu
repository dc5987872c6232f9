// libsa_b200.so -- host side of the C ABI declared in include/sa_api.h.
// Owns: scratch for the per-CTA candidate lists, pinned staging, TMA descriptors, CUDA events.
// Never owns or copies the corpus.  No CPU fallback anywhere: every entry point ends in a kernel launch.
#include "../../include/sa_api.h"
#include "sa_aux.cuh"
#include "sa_scan.cuh"

#include <cuda.h>
#include <cuda_runtime.h>
#include <dlfcn.h>
#include <nccl.h>  // types and prototypes only: the library itself is dlopen'ed (sa_comm_*), never linked

#include <algorithm>
#include <climits>
#include <cstdarg>
#include <cstddef>
#include <cstdio>
#include <cstring>
#include <string>
#include <vector>

namespace {

thread_local char g_err[512] = "";

int vfail(int rc, const char* fmt, va_list ap) {
  vsnprintf(g_err, sizeof g_err, fmt, ap);
  return rc;
}

int fail(int rc, const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vfail(rc, fmt, ap);
  va_end(ap);
  return rc;
}

}  // namespace

// used by the other translation units of the library (sa_wire.cpp); not part of the public headers
extern "C" int sa_internal_fail(int rc, const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vfail(rc, fmt, ap);
  va_end(ap);
  return rc;
}

namespace {

#define SA_CUDA(call)                                                                                \
  do {                                                                                               \
    cudaError_t _e = (call);                                                                         \
    if (_e != cudaSuccess)                                                                           \
      return fail(SA_ERR_CUDA, "%s failed: %s (%s:%d)", #call, cudaGetErrorString(_e), __FILE__, __LINE__); \
  } while (0)

using EncodeTiledFn = CUresult (*)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                   const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                   CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

EncodeTiledFn get_encode_fn() {
  static EncodeTiledFn fn = nullptr;
  if (fn) return fn;
  void* p = nullptr;
  cudaDriverEntryPointQueryResult qres;
  if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) != cudaSuccess ||
      qres != cudaDriverEntryPointSuccess)
    return nullptr;
  fn = reinterpret_cast<EncodeTiledFn>(p);
  return fn;
}

// 2-D tensor [rows x dim] of the engine's element type, box = one 128-B K slice (SWIZZLE_128B: 64 bf16 or 128 int8
// columns) x box_rows rows.
int encode_rows_map(CUtensorMap* m, const void* base, uint64_t rows, int dim, int box_rows, int elem) {
  EncodeTiledFn fn = get_encode_fn();
  if (!fn) return fail(SA_ERR_CUDA, "cuTensorMapEncodeTiled entry point not available");
  const bool i8 = elem == SA_ELEM_INT8;
  cuuint64_t gdim[2] = {static_cast<cuuint64_t>(dim), rows};
  cuuint64_t gstride[1] = {static_cast<cuuint64_t>(dim) * sa::elem_bytes(elem)};
  cuuint32_t box[2] = {static_cast<cuuint32_t>(i8 ? sa::kBlockKI8 : sa::kBlockK), static_cast<cuuint32_t>(box_rows)};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = fn(m, i8 ? CU_TENSOR_MAP_DATA_TYPE_UINT8 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(base), gdim, gstride, box, estr,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return fail(SA_ERR_CUDA, "cuTensorMapEncodeTiled failed with CUresult %d", (int)r);
  return SA_OK;
}

// Entry points switch to the engine's device and switch back on return, so a caller driving several GPUs from one
// thread keeps its own current device.
struct DeviceGuard {
  int prev = -1;
  cudaError_t rc = cudaSuccess;
  explicit DeviceGuard(int dev) {
    rc = cudaGetDevice(&prev);
    if (rc == cudaSuccess && prev != dev) rc = cudaSetDevice(dev);
    else if (rc == cudaSuccess) prev = -1;  // nothing to restore
  }
  ~DeviceGuard() {
    if (prev >= 0) cudaSetDevice(prev);
  }
};
#define SA_ON_DEVICE(dev)                                                                             \
  DeviceGuard _dg(dev);                                                                              \
  if (_dg.rc != cudaSuccess) return fail(SA_ERR_CUDA, "cudaSetDevice(%d) failed: %s", (dev), cudaGetErrorString(_dg.rc))

constexpr int kMaxLaunches = 16;
constexpr int kDefaultWaitHintNs = 0;  // plain polling (option "wait_hint_ns" overrides)
constexpr int kDefaultPresample = 0;   // no sampling pre-pass (option "presample" overrides)
constexpr int kTimingRing = 16;
constexpr int kHostSlots = SA_HOST_SLOTS;

}  // namespace

struct sa_engine {
  int device = 0;
  int dim = 0;
  int64_t capacity = 0;
  int max_batch = 0;
  int max_k = 0;
  int num_sms = 0;
  int sim = SA_SIM_COSINE;     // fixed at creation
  int elem = SA_ELEM_BF16;     // fixed at creation: the element type of the rows and of the device queries

  void* corpus = nullptr;      // caller-owned [capacity][dim] of elem
  float* row_term = nullptr;   // caller-owned: 1/|c| (cosine), 1 (dotProduct), |c|^2/2 (euclidean); see sa_aux.cuh
  unsigned* cmax = nullptr;    // device scalar (float bits): upper bound on |c| over the committed rows (not cosine)
  unsigned long long* row_tags = nullptr;  // caller-owned [capacity] filter tags (sa_corpus_bind_tags), or nullptr
  int64_t n_rows = 0;
  CUtensorMap tmap_c[2];       // [0]: box 256 rows (cta_group 1), [1]: box 128 rows (cta_group 2, multicast)
  bool bound = false;

  // scratch (library-owned)
  float* part_score = nullptr;  // [num_sms][128][32]
  int* part_idx = nullptr;
  float* part_drop = nullptr;   // [num_sms][128]
  double* res64 = nullptr;      // [max_batch][max_k] internal result of a search: value (float64, larger is better) ...
  int* residx = nullptr;        // ... and shard-local row
  sa::FixEntry* fix_entries = nullptr;  // [kMaxLaunches * num_sms * 128] work queue of the exact fallback scan
  sa::FixQuery* fix_query = nullptr;    // [max_batch]
  int* fix_counters = nullptr;          // [0] queue length, [1] CTAs done (both zero between searches)
  uint16_t* q_bf16 = nullptr;   // [max_batch][dim] converted queries: bf16, or int8 bytes in the same buffer
  float* q_f32 = nullptr;       // [max_batch][dim]  (host-path staging on device)
  float* res_score = nullptr;   // [max_batch][max_k]
  int* res_idx = nullptr;
  sa::PackedHit* hits = nullptr;  // [max_batch][max_k] this shard's (cosine f64, global row) lists for the exchange
  long long* res_row64 = nullptr; // [max_batch][max_k] merged global rows (sharded host path)
  // host-buffer path: pinned staging per slot (0,1 = public asynchronous slots, 2 = the blocking sa_search_host)
  struct HostSlot {
    float* h_q = nullptr;      // pinned [max_batch][dim]
    float* h_score = nullptr;  // pinned [max_batch][max_k]
    int* h_idx = nullptr;      // pinned
    long long* h_row64 = nullptr;  // pinned [max_batch][max_k] (sharded searches return global rows)
    sa::Filter* h_f = nullptr;     // pinned [max_batch] filters of a filtered search ...
    sa::Filter* d_f = nullptr;     // ... and their device copy
    bool sharded = false;
    cudaEvent_t done = nullptr;
    int nq = 0, k = 0;
    bool busy = false;
  };
  HostSlot slot[kHostSlots + 1];
  float* d_stage = nullptr;     // device staging for host ingest
  float* h_stage = nullptr;     // pinned staging for host ingest
  int64_t stage_rows = 0;
  cudaStream_t own_stream = nullptr;
  cudaEvent_t scratch_free = nullptr;  // recorded after every search: the scratch buffers are shared by all searches

  long long* dbg_times = nullptr;  // [num_sms][2] CTA start/end timestamps of the last scan launch (option "record_times")
  int opt_record_times = 0;
  sa::ScanProf* prof = nullptr;    // [num_sms] per-CTA role counters of the last scan launch (option "profile")
  int opt_profile = 0;
  int last_grid = 0;
  // Shared per-query thresholds [thr_n] and drift counters [kMaxLaunches * num_sms] of the scan.  Both must be zero when
  // a scan starts; every scan launch of a search uses its own slice and the search's last kernel re-zeroes what was used.
  unsigned* thr_shared = nullptr;
  int thr_n = 0;
  int* lane_progress = nullptr;
  unsigned* lane2 = nullptr;  // [kMaxLaunches][num_sms * 128] the lanes' second-best scores (window bound); zero like the above
  bool scratch_dirty = false;  // a search failed between its first launch and its last: re-zero before the next one
  int opt_share_thresholds = 1;
  int opt_window_bound = 1;

  // options
  int opt_cta_group = 0;
  int opt_max_launch_qblocks = 0;
  int opt_max_drift = -1;  // -1 = auto (1 tile)
  int opt_pace_gain = -1;  // -1 = auto (128 cycles/tile for CTA pairs, 64 for single CTAs), 0 = off
  int opt_pace_max = -1;   // -1 = auto (8 x gain)
  int opt_unit_map = 0;
  int opt_list_len = 0;    // 0 = auto (16 when k <= 16, else 32)
  int opt_wait_hint_ns = -1;  // suspend-time hint of the epilogue's mbarrier waits (-1 = auto, 0 = plain polling)
  int opt_presample = -1;  // tile stride of the sampling pre-pass that seeds the shared thresholds (-1 = auto, 0 = off)
  int opt_force_fix = 0;   // test hook: every (query, lane) goes through the exact fallback scan
  int64_t last_fix_entries = -1;  // option "count_fix": work-queue length of the last search (costs a host sync)
  int opt_count_fix = 0;

  // timing: CUDA events of the most recent kTimingRing searches
  struct Timing {
    cudaEvent_t ev_total[2] = {nullptr, nullptr};
    cudaEvent_t ev_scan[kMaxLaunches][2];
    int launches = 0;
    int kernels = 0;
    double bytes = 0, flops = 0;
  };
  Timing ring[kTimingRing];
  long long n_searches = 0;
};

namespace {

// asc = 1: the hits are Euclidean distances (smaller is better)
int launch_merge_packed(const sa::PackedHit* hits, int n_shards, int nq, int k, float* out_score, long long* out_row,
                        int asc, cudaStream_t st) {
  if (n_shards <= 32 && n_shards * k <= 256 && k <= sa::kMergePackedMaxK)
    sa::sa_merge_packed_kernel<<<(nq + sa::kMergePackedWarps - 1) / sa::kMergePackedWarps, sa::kMergePackedWarps * 32, 0, st>>>(
        hits, n_shards, nq, k, out_score, out_row, asc);
  else
    sa::sa_merge_serial_kernel<<<(nq + 127) / 128, 128, 0, st>>>(sa::PackedHits{hits}, n_shards, nq, k, out_score,
                                                                  out_row, asc);
  SA_CUDA(cudaGetLastError());
  return SA_OK;
}

struct LaunchPlan {
  int cg;
  int q0;   // first query of this launch
  int nq;   // queries in this launch
  int nqb;  // query blocks (of 128*cg)
  int tl;   // tile lanes
};

// Tile lanes and walk length of one launch holding `per` query blocks.
void lanes_for(int units, int per, int num_tiles, int* tl, long* cost) {
  const int tl1 = std::max(1, std::min(std::min(units / per, num_tiles), sa::kMaxLanes));
  *tl = tl1;
  *cost = (num_tiles + tl1 - 1) / tl1;
}

// Split the batch into scan launches.  A launch with nqb query blocks runs TL = floor(units / nqb) tile
// lanes, each walking ceil(num_tiles / TL) tiles; pick the split that minimises the summed tile walks
// (fewer launches win ties: every launch re-streams the corpus through HBM once).
std::vector<LaunchPlan> plan_search(int num_sms, int max_launch_qblocks, int nq, int cg, int num_tiles) {
  const int rows_per_qb = 128 * cg;
  const int units = num_sms / cg;
  const int nqb_total = (nq + rows_per_qb - 1) / rows_per_qb;
  int cap = units;
  if (max_launch_qblocks > 0) cap = std::min(cap, max_launch_qblocks);
  long best_cost = -1;
  int best_l = 1;
  const int l_min = (nqb_total + cap - 1) / cap;
  for (int l = l_min; l <= std::min(nqb_total, l_min + 7); ++l) {
    long cost = 0;
    int left = nqb_total;
    for (int i = 0; i < l; ++i) {
      const int per = (left + (l - i) - 1) / (l - i);
      int tl;
      long c;
      lanes_for(units, per, num_tiles, &tl, &c);
      cost += c;
      left -= per;
    }
    if (best_cost < 0 || cost * 100 < best_cost * 97) {  // a later (more launches) split must win by > 3 %
      best_cost = cost;
      best_l = l;
    }
  }
  std::vector<LaunchPlan> out;
  int left = nqb_total, qb0 = 0;
  for (int i = 0; i < best_l; ++i) {
    const int per = (left + (best_l - i) - 1) / (best_l - i);
    LaunchPlan lp;
    long c;
    lp.cg = cg;
    lp.q0 = qb0 * rows_per_qb;
    lp.nq = std::min(nq - lp.q0, per * rows_per_qb);
    lp.nqb = per;
    lanes_for(units, per, num_tiles, &lp.tl, &c);
    out.push_back(lp);
    qb0 += per;
    left -= per;
  }
  return out;
}

template <int kCG, int kKL, int kMode, int kEpi>
int launch_scan(const CUtensorMap& tq, const CUtensorMap& tc, const sa::ScanParams& p, int grid, cudaStream_t st) {
  auto kern = sa::sa_scan_kernel<kCG, kKL, kMode, kEpi>;
  constexpr uint32_t kSmem = sa::ScanCfg<kCG, (kEpi & sa::kEpiFilt) != 0>::kSmemBytes;
  // per-device attribute; a few microseconds, so set it on every launch rather than caching per device
  SA_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmem));
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(grid);
  cfg.blockDim = dim3(sa::kScanThreads);
  cfg.dynamicSmemBytes = kSmem;
  cfg.stream = st;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeClusterDimension;
  attr[0].val.clusterDim.x = kCG;
  attr[0].val.clusterDim.y = 1;
  attr[0].val.clusterDim.z = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  SA_CUDA(cudaLaunchKernelEx(&cfg, kern, tq, tc, p));
  return SA_OK;
}

// Every instantiation of the scan kernel, one row each: {cta_group, list length, build, epilogue, launcher}.
// epi: sa::kEpiMul (cosine, dotProduct) or sa::kEpiSub (euclidean), | sa::kEpiFilt for a filtered search,
// | sa::kEpiDeep for a deep search (k > 28, 32-entry lists).  Filtered and deep searches have the production build
// only; the profiling build has 16-entry lists only; the debug dump reads raw accumulators, which do not depend on the
// epilogue, so it has the multiply form only.
using ScanLauncher = int (*)(const CUtensorMap&, const CUtensorMap&, const sa::ScanParams&, int, cudaStream_t);
struct ScanVariant {
  int cg, kl, mode, epi;
  ScanLauncher launch;
};
constexpr int kProd = sa::kModeProd, kProf = sa::kModeProf, kDots = sa::kModeDots;
constexpr int kMul = sa::kEpiMul, kSub = sa::kEpiSub, kFilt = sa::kEpiFilt, kDeep = sa::kEpiDeep, kI8 = sa::kEpiI8;
constexpr ScanVariant kScanVariants[] = {
    // production
    {1, 16, kProd, kMul, &launch_scan<1, 16, kProd, kMul>},
    {1, 32, kProd, kMul, &launch_scan<1, 32, kProd, kMul>},
    {2, 16, kProd, kMul, &launch_scan<2, 16, kProd, kMul>},
    {2, 32, kProd, kMul, &launch_scan<2, 32, kProd, kMul>},
    {1, 16, kProd, kSub, &launch_scan<1, 16, kProd, kSub>},
    {1, 32, kProd, kSub, &launch_scan<1, 32, kProd, kSub>},
    {2, 16, kProd, kSub, &launch_scan<2, 16, kProd, kSub>},
    {2, 32, kProd, kSub, &launch_scan<2, 32, kProd, kSub>},
    {1, 16, kProd, kMul | kFilt, &launch_scan<1, 16, kProd, kMul | kFilt>},
    {1, 32, kProd, kMul | kFilt, &launch_scan<1, 32, kProd, kMul | kFilt>},
    {2, 16, kProd, kMul | kFilt, &launch_scan<2, 16, kProd, kMul | kFilt>},
    {2, 32, kProd, kMul | kFilt, &launch_scan<2, 32, kProd, kMul | kFilt>},
    {1, 16, kProd, kSub | kFilt, &launch_scan<1, 16, kProd, kSub | kFilt>},
    {1, 32, kProd, kSub | kFilt, &launch_scan<1, 32, kProd, kSub | kFilt>},
    {2, 16, kProd, kSub | kFilt, &launch_scan<2, 16, kProd, kSub | kFilt>},
    {2, 32, kProd, kSub | kFilt, &launch_scan<2, 32, kProd, kSub | kFilt>},
    // deep
    {1, 32, kProd, kMul | kDeep, &launch_scan<1, 32, kProd, kMul | kDeep>},
    {2, 32, kProd, kMul | kDeep, &launch_scan<2, 32, kProd, kMul | kDeep>},
    {1, 32, kProd, kSub | kDeep, &launch_scan<1, 32, kProd, kSub | kDeep>},
    {2, 32, kProd, kSub | kDeep, &launch_scan<2, 32, kProd, kSub | kDeep>},
    {1, 32, kProd, kMul | kFilt | kDeep, &launch_scan<1, 32, kProd, kMul | kFilt | kDeep>},
    {2, 32, kProd, kMul | kFilt | kDeep, &launch_scan<2, 32, kProd, kMul | kFilt | kDeep>},
    {1, 32, kProd, kSub | kFilt | kDeep, &launch_scan<1, 32, kProd, kSub | kFilt | kDeep>},
    {2, 32, kProd, kSub | kFilt | kDeep, &launch_scan<2, 32, kProd, kSub | kFilt | kDeep>},
    // profiling
    {1, 16, kProf, kMul, &launch_scan<1, 16, kProf, kMul>},
    {2, 16, kProf, kMul, &launch_scan<2, 16, kProf, kMul>},
    {1, 16, kProf, kSub, &launch_scan<1, 16, kProf, kSub>},
    {2, 16, kProf, kSub, &launch_scan<2, 16, kProf, kSub>},
    // debug dots
    {1, 16, kDots, kMul, &launch_scan<1, 16, kDots, kMul>},
    {2, 16, kDots, kMul, &launch_scan<2, 16, kDots, kMul>},
    // int8 index: the same rows | kI8
    {1, 16, kProd, kMul | kI8, &launch_scan<1, 16, kProd, kMul | kI8>},
    {1, 32, kProd, kMul | kI8, &launch_scan<1, 32, kProd, kMul | kI8>},
    {2, 16, kProd, kMul | kI8, &launch_scan<2, 16, kProd, kMul | kI8>},
    {2, 32, kProd, kMul | kI8, &launch_scan<2, 32, kProd, kMul | kI8>},
    {1, 16, kProd, kSub | kI8, &launch_scan<1, 16, kProd, kSub | kI8>},
    {1, 32, kProd, kSub | kI8, &launch_scan<1, 32, kProd, kSub | kI8>},
    {2, 16, kProd, kSub | kI8, &launch_scan<2, 16, kProd, kSub | kI8>},
    {2, 32, kProd, kSub | kI8, &launch_scan<2, 32, kProd, kSub | kI8>},
    {1, 16, kProd, kMul | kFilt | kI8, &launch_scan<1, 16, kProd, kMul | kFilt | kI8>},
    {1, 32, kProd, kMul | kFilt | kI8, &launch_scan<1, 32, kProd, kMul | kFilt | kI8>},
    {2, 16, kProd, kMul | kFilt | kI8, &launch_scan<2, 16, kProd, kMul | kFilt | kI8>},
    {2, 32, kProd, kMul | kFilt | kI8, &launch_scan<2, 32, kProd, kMul | kFilt | kI8>},
    {1, 16, kProd, kSub | kFilt | kI8, &launch_scan<1, 16, kProd, kSub | kFilt | kI8>},
    {1, 32, kProd, kSub | kFilt | kI8, &launch_scan<1, 32, kProd, kSub | kFilt | kI8>},
    {2, 16, kProd, kSub | kFilt | kI8, &launch_scan<2, 16, kProd, kSub | kFilt | kI8>},
    {2, 32, kProd, kSub | kFilt | kI8, &launch_scan<2, 32, kProd, kSub | kFilt | kI8>},
    {1, 32, kProd, kMul | kDeep | kI8, &launch_scan<1, 32, kProd, kMul | kDeep | kI8>},
    {2, 32, kProd, kMul | kDeep | kI8, &launch_scan<2, 32, kProd, kMul | kDeep | kI8>},
    {1, 32, kProd, kSub | kDeep | kI8, &launch_scan<1, 32, kProd, kSub | kDeep | kI8>},
    {2, 32, kProd, kSub | kDeep | kI8, &launch_scan<2, 32, kProd, kSub | kDeep | kI8>},
    {1, 32, kProd, kMul | kFilt | kDeep | kI8, &launch_scan<1, 32, kProd, kMul | kFilt | kDeep | kI8>},
    {2, 32, kProd, kMul | kFilt | kDeep | kI8, &launch_scan<2, 32, kProd, kMul | kFilt | kDeep | kI8>},
    {1, 32, kProd, kSub | kFilt | kDeep | kI8, &launch_scan<1, 32, kProd, kSub | kFilt | kDeep | kI8>},
    {2, 32, kProd, kSub | kFilt | kDeep | kI8, &launch_scan<2, 32, kProd, kSub | kFilt | kDeep | kI8>},
    {1, 16, kProf, kMul | kI8, &launch_scan<1, 16, kProf, kMul | kI8>},
    {2, 16, kProf, kMul | kI8, &launch_scan<2, 16, kProf, kMul | kI8>},
    {1, 16, kDots, kMul | kI8, &launch_scan<1, 16, kDots, kMul | kI8>},
    {2, 16, kDots, kMul | kI8, &launch_scan<2, 16, kDots, kMul | kI8>},
};

int launch_scan_dispatch(int cg, int kl, int mode, int epi, const CUtensorMap& tq, const CUtensorMap& tc,
                         const sa::ScanParams& p, int grid, cudaStream_t st) {
  for (const ScanVariant& v : kScanVariants)
    if (v.cg == cg && v.kl == kl && v.mode == mode && v.epi == epi) return v.launch(tq, tc, p, grid, st);
  static const char* const kBuild[] = {"production", "debug-dots", "profiling"};  // indexed by sa::kMode*
  return fail(SA_ERR_ARG, "no scan instantiation for cta_group %d, %d-entry lists, %s build, %s%s%s%s epilogue", cg, kl,
              kBuild[mode], (epi & kSub) ? "subtract" : "multiply", (epi & kFilt) ? " filtered" : "",
              (epi & kDeep) ? " deep" : "", (epi & kI8) ? " int8" : "");
}

int choose_cg(const sa_engine* e, int nq) {
  if (e->opt_cta_group == 1 || e->opt_cta_group == 2) return e->opt_cta_group;
  // Auto: a CTA pair shares the corpus tile between two query blocks (each corpus slice is read from L2 once and
  // multicast to both), which pays once the batch fills 256-row pair blocks; small batches are HBM-bound and use 1 CTA.
  return nq > 128 ? 2 : 1;
}

bool is_pinned(const void* p) {
  cudaPointerAttributes a;
  if (cudaPointerGetAttributes(&a, p) != cudaSuccess) {
    cudaGetLastError();  // clear the sticky "invalid value" some drivers report for plain malloc memory
    return false;
  }
  return a.type == cudaMemoryTypeHost;
}

int check_engine(const sa_engine* e) {
  if (!e) return fail(SA_ERR_ARG, "null engine");
  if (!e->bound) return fail(SA_ERR_ARG, "no corpus bound (call sa_corpus_bind)");
  return SA_OK;
}

// The scan's approximate score a = fp32_accumulate(q . c) * fl(1/|c|) against the exact e = <q, c>/|c|, both divided by
// |q|:  fp32 accumulation of dim exact products, each addition off by at most one ulp of the running magnitude
// (<= |q||c| by Cauchy-Schwarz): dim * 2^-23;  the inverse norm (fp32 sum of squares over dim/32 terms per lane + a
// 5-level butterfly, one square root, one division) and the final multiply: (dim/64 + 6) * 2^-23, rounded up generously.
// Measured worst case on adversarial inputs is ~100x smaller (tests/test_gpu_parity.py::test_scan_error_is_inside_eps).
// int8: the accumulator is the exact integer <q,c>, so only its conversion to fp32 (2^-24 |<q,c>|), the row term's one
// rounding (2^-24) and the final multiply (2^-24) remain: 3 * 2^-24 relative (cosine), rounded up to 4 * 2^-23 whatever
// the dim.  The euclidean subtraction and its row term are covered by cert_eps's own 2^-23 terms (DESIGN.md section 4.2).
constexpr float kScanEpsRelI8 = 4.0f * 1.1920929e-07f;
float scan_eps_rel(int dim, int elem) {
  return elem == SA_ELEM_INT8 ? kScanEpsRelI8 : (1.0625f * dim + 16.0f) * 1.1920929e-07f;
}

int zero_scan_scratch(sa_engine* e, cudaStream_t st) {
  SA_CUDA(cudaMemsetAsync(e->thr_shared, 0, sizeof(unsigned) * e->thr_n, st));
  SA_CUDA(cudaMemsetAsync(e->lane_progress, 0, sizeof(int) * kMaxLaunches * e->num_sms, st));
  SA_CUDA(cudaMemsetAsync(e->lane2, 0, sizeof(unsigned) * kMaxLaunches * e->num_sms * 128, st));
  SA_CUDA(cudaMemsetAsync(e->fix_counters, 0, sizeof(int) * 2, st));
  return SA_OK;
}

// A filtered search needs its filters and a bound tag array.
int check_filtered(const sa_engine* e, const void* filters) {
  if (!filters) return fail(SA_ERR_ARG, "null filters");
  if (!e->row_tags) return fail(SA_ERR_ARG, "filtered search without row tags (call sa_corpus_bind_tags)");
  return SA_OK;
}

// The first checks of a search entry point; `filtered`: the filtered twin, which refuses null filters.  The order
// matters: check_filtered reads the engine, and a sharded search must report an argument error before check_rank_comm,
// whose first call on a communicator is a collective.
int check_search(const sa_engine* e, const void* filters, bool filtered) {
  int rc = check_engine(e);
  if (rc == SA_OK && filtered) rc = check_filtered(e, filters);
  return rc;
}

// fp32 queries -> the engine's element type in the query scratch (int8: f32_to_i8, the bytes of the same buffer)
int convert_queries(sa_engine* e, const float* q_f32_dev, int nq, cudaStream_t st) {
  SA_CUDA(cudaStreamWaitEvent(st, e->scratch_free, 0));  // q_bf16 is scratch too: the previous search still reads it
  const long long threads = static_cast<long long>(nq) * 32;
  const unsigned grid = static_cast<unsigned>((threads + 255) / 256);
  if (e->elem == SA_ELEM_INT8)
    sa::sa_convert_rows_i8_kernel<<<grid, 256, 0, st>>>(q_f32_dev, reinterpret_cast<int8_t*>(e->q_bf16), nullptr, nq,
                                                        e->dim, e->sim, nullptr);
  else
    sa::sa_convert_rows_kernel<<<grid, 256, 0, st>>>(q_f32_dev, e->q_bf16, nullptr, nq, e->dim);
  SA_CUDA(cudaGetLastError());
  return SA_OK;
}

// One search = per scan launch {scan kernel, merge/certify kernel}, then one fixup kernel (exact fallback scan of the
// ambiguous (query, lane) pairs -- normally none -- and conversion of the internal result to the caller's arrays).
// filters (device, [nq]) != nullptr: a filtered search; every kernel sees only the rows that pass each query's filter.
int do_search(sa_engine* e, const void* q_dev, int nq, int k, float* out_score, int32_t* out_idx,
              double* out_score64, sa::PackedHit* out_packed, int64_t row_offset, cudaStream_t st,
              const sa::Filter* filters = nullptr) {
  if (nq <= 0 || nq > e->max_batch) return fail(SA_ERR_CAPACITY, "nq %d outside [1, max_batch %d]", nq, e->max_batch);
  if (k <= 0 || k > e->max_k) return fail(SA_ERR_ARG, "k %d outside [1, max_k %d]", k, e->max_k);
  if (!q_dev || !out_score || !out_idx) return fail(SA_ERR_ARG, "null buffer");
  if (reinterpret_cast<uintptr_t>(q_dev) % 16) return fail(SA_ERR_ARG, "query buffer must be 16-byte aligned");
  SA_ON_DEVICE(e->device);

  // 16-entry lists for k <= 16: with the certificate any k <= kKL is exact; a margin of spare entries only makes the
  // fallback rarer, and it is already rare once a tile lane holds more than a few thousand rows.  A deep search
  // (k > 28) keeps the 32-entry lists and runs the scan variant whose shared bounds hold for its k (sa_scan.cuh,
  // kEpiDeep): the certificate needs k <= |U|, not k <= kKL.
  const int kl = e->opt_list_len ? e->opt_list_len : (k <= 16 ? 16 : 32);
  const bool deep = k > sa::kShallowMaxK;
  if (k > (kl == 32 ? SA_MAX_K : kl)) return fail(SA_ERR_ARG, "k %d needs candidate lists longer than list_len %d", k, kl);
  const int64_t n_rows = e->n_rows;
  const int num_tiles = static_cast<int>((n_rows + sa::kBlockN - 1) / sa::kBlockN);
  const int cg = choose_cg(e, nq);
  std::vector<LaunchPlan> plan = plan_search(e->num_sms, e->opt_max_launch_qblocks, nq, cg, std::max(num_tiles, 1));
  if (static_cast<int>(plan.size()) > kMaxLaunches)
    return fail(SA_ERR_CAPACITY, "batch needs %zu scan launches (max %d)", plan.size(), kMaxLaunches);
  const int mode = e->opt_profile ? sa::kModeProf : sa::kModeProd;
  const int epi = (e->sim == SA_SIM_EUCLIDEAN ? sa::kEpiSub : sa::kEpiMul) | (filters != nullptr ? sa::kEpiFilt : 0) |
                  (deep ? sa::kEpiDeep : 0) | (e->elem == SA_ELEM_INT8 ? sa::kEpiI8 : 0);
  const float eps_rel = scan_eps_rel(e->dim, e->elem);
  const size_t row_bytes = static_cast<size_t>(e->dim) * sa::elem_bytes(e->elem);

  // The candidate lists, shared thresholds and drift counters are one set of scratch buffers: a search issued on
  // another stream than the previous one must not start before that one has finished with them.
  SA_CUDA(cudaStreamWaitEvent(st, e->scratch_free, 0));
  if (e->scratch_dirty) {
    int rc = zero_scan_scratch(e, st);
    if (rc) return rc;
    e->scratch_dirty = false;
  }
  sa_engine::Timing& tm = e->ring[e->n_searches % kTimingRing];
  tm.launches = 0;
  tm.kernels = 0;
  SA_CUDA(cudaEventRecord(tm.ev_total[0], st));
  e->scratch_dirty = true;  // cleared again once the fixup kernel (which re-zeroes the scratch) is enqueued
  int min_tl = sa::kMaxLanes;
  for (size_t li = 0; li < plan.size(); ++li) {
    const LaunchPlan& lp = plan[li];
    const void* qptr = static_cast<const char*>(q_dev) + lp.q0 * row_bytes;
    CUtensorMap tq;
    int rc = encode_rows_map(&tq, qptr, static_cast<uint64_t>(lp.nq), e->dim, sa::kBlockM, e->elem);
    if (rc) return rc;

    sa::ScanParams sp = {};
    sp.row_term = e->row_term;
    sp.n_rows = n_rows;
    sp.nq = lp.nq;
    sp.num_kb = static_cast<int>(row_bytes / 128);  // 128-byte K slices
    sp.num_tiles = num_tiles;
    sp.nqb = lp.nqb;
    sp.tl_count = lp.tl;
    sp.part_score = e->part_score;
    sp.part_idx = e->part_idx;
    sp.part_drop = e->part_drop;
    sp.corpus_evict_first = (lp.nqb == 1) ? 1 : 0;  // a tile nobody else will ask for: stream it through L2
    sp.tile_stride = 1;
    sp.wait_hint_ns = e->opt_wait_hint_ns >= 0 ? e->opt_wait_hint_ns : kDefaultWaitHintNs;
    sp.lane_progress = nullptr;
    sp.max_drift = e->opt_max_drift >= 0 ? e->opt_max_drift : 1;
    sp.pace_gain = 0;
    sp.unit_map = e->opt_unit_map;
    // drift-control defaults: one tile of free lead, then 64 (single CTAs) or 128 (pairs) cycles of delay per K-slice
    // issue per extra tile of lead (a tile is num_kb K slices); options "max_drift", "pace_gain" and "pace_max"
    // override them
    const int gain = e->opt_pace_gain >= 0 ? e->opt_pace_gain : (lp.cg == 2 ? 128 : 64);
    sp.pace_max = e->opt_pace_max >= 0 ? e->opt_pace_max : 8 * gain;
    if (lp.nqb > 1 && gain > 0) {
      sp.lane_progress = e->lane_progress + li * e->num_sms;  // this launch's slice (zero: see sa_engine)
      sp.pace_gain = gain;
    }
    const int presample = e->opt_presample >= 0 ? e->opt_presample : kDefaultPresample;
    // a pre-pass only pays when every lane still has a long walk ahead of it after the sample
    const bool do_presample = presample > 1 && e->opt_share_thresholds && num_tiles >= 4 * presample * lp.tl;
    sp.thr_shared = (e->opt_share_thresholds && (lp.tl > 1 || do_presample)) ? e->thr_shared + lp.q0 : nullptr;
    // window bound: lp.tl * lp.nqb * 128 * lp.cg <= num_sms * 128 slots, this launch's slice of the table
    sp.lane2 = (sp.thr_shared != nullptr && e->opt_window_bound && lp.tl >= sa::kWin)
                   ? e->lane2 + static_cast<size_t>(li) * e->num_sms * 128 : nullptr;
    sp.dbg_dots = nullptr;
    sp.dbg_tile = -1;
    sp.dbg_times = e->opt_record_times ? e->dbg_times : nullptr;
    sp.prof = e->prof;
    if (filters != nullptr) {
      sp.row_tags = e->row_tags;
      sp.filters = filters + lp.q0;
    }
    const int grid = lp.nqb * lp.tl * lp.cg;
    e->last_grid = grid;
    min_tl = std::min(min_tl, lp.tl);

    sa::MergeParams mp = {};
    mp.part_score = e->part_score;
    mp.part_idx = e->part_idx;
    mp.part_drop = e->part_drop;
    mp.corpus = e->corpus;
    mp.queries = qptr;
    mp.dim = e->dim;
    mp.nq = lp.nq;
    mp.k = k;
    mp.cg = lp.cg;
    mp.nqb = lp.nqb;
    mp.tl_count = lp.tl;
    mp.unit_map = e->opt_unit_map;
    mp.q0 = lp.q0;
    mp.eps_rel = eps_rel;
    mp.sim = e->sim;
    mp.elem = e->elem;
    mp.cmax = e->cmax;
    mp.res64 = e->res64 + static_cast<size_t>(lp.q0) * k;
    mp.residx = e->residx + static_cast<size_t>(lp.q0) * k;
    mp.fix_entries = e->fix_entries;
    mp.fix_count = e->fix_counters;
    mp.fix_query = e->fix_query;
    mp.force_fix = e->opt_force_fix;

    SA_CUDA(cudaEventRecord(tm.ev_scan[li][0], st));
    if (do_presample) {
      // Sampling pre-pass: the same kernel over every presample-th tile, then each query's kKL-th best of the sample
      // becomes its shared threshold (a valid lower bound on its global kKL-th best; a deep search: its k-th best, a
      // bound on the global k-th best, and the only seed its shared threshold gets).  The full scan then starts with
      // thresholds near their final values whatever the order of the rows: an adversarial (e.g. ascending) order can no
      // longer make every row an insertion.
      sa::ScanParams pp = sp;
      pp.tile_stride = presample;
      pp.lane_progress = nullptr;  // no pacing: the pre-pass is short
      pp.pace_gain = 0;
      pp.lane2 = nullptr;
      pp.prof = e->prof;
      rc = launch_scan_dispatch(lp.cg, kl, sa::kModeProd, epi, tq, e->tmap_c[lp.cg - 1], pp, grid, st);
      if (rc) return rc;
      sa::MergeParams bp = mp;  // with bound_out set the merge kernel publishes the bounds and reads no result field
      bp.bound_out = e->thr_shared + lp.q0;
      if (kl == 16)
        sa::sa_merge_rescore_kernel<16><<<lp.nq, sa::kMergeThreads, 0, st>>>(bp);
      else
        sa::sa_merge_rescore_kernel<32><<<lp.nq, sa::kMergeThreads, 0, st>>>(bp);
      SA_CUDA(cudaGetLastError());
      tm.kernels += 2;
    }
    rc = launch_scan_dispatch(lp.cg, kl, mode, epi, tq, e->tmap_c[lp.cg - 1], sp, grid, st);
    if (rc) return rc;
    SA_CUDA(cudaEventRecord(tm.ev_scan[li][1], st));
    if (kl == 16)
      sa::sa_merge_rescore_kernel<16><<<lp.nq, sa::kMergeThreads, 0, st>>>(mp);
    else
      sa::sa_merge_rescore_kernel<32><<<lp.nq, sa::kMergeThreads, 0, st>>>(mp);
    SA_CUDA(cudaGetLastError());
    tm.launches += 1;
    tm.kernels += 2;
  }
  if (e->opt_count_fix) {
    int cnt = 0;
    SA_CUDA(cudaMemcpyAsync(&cnt, e->fix_counters, sizeof(int), cudaMemcpyDeviceToHost, st));
    SA_CUDA(cudaStreamSynchronize(st));
    e->last_fix_entries = cnt;
  }
  {
    sa::FixParams fp = {};
    fp.entries = e->fix_entries;
    fp.fix_count = e->fix_counters;
    fp.done_count = e->fix_counters + 1;
    fp.fix_query = e->fix_query;
    fp.corpus = e->corpus;
    fp.row_term = e->row_term;
    fp.queries = q_dev;
    fp.n_rows = n_rows;
    fp.num_tiles = num_tiles;
    fp.dim = e->dim;
    fp.nq = nq;
    fp.k = k;
    const int tiles_per_lane = (std::max(num_tiles, 1) + min_tl - 1) / min_tl;
    fp.chunks_per_entry = (tiles_per_lane + sa::kFixChunkTiles - 1) / sa::kFixChunkTiles;
    fp.sim = e->sim;
    fp.elem = e->elem;
    fp.res64 = e->res64;
    fp.residx = e->residx;
    fp.out_score = out_score;
    fp.out_idx = out_idx;
    fp.out_score64 = out_score64;
    fp.out_packed = out_packed;
    fp.row_offset = row_offset;
    fp.zero_a = e->thr_shared;
    fp.zero_a_n = std::min(e->thr_n, ((nq + 255) / 256) * 256);
    fp.zero_b = e->lane_progress;
    fp.zero_b_n = static_cast<int>(plan.size()) * e->num_sms;
    fp.zero_c = e->lane2;
    fp.zero_c_n = e->opt_window_bound ? static_cast<int>(plan.size()) * e->num_sms * 128 : 0;
    fp.row_tags = filters != nullptr ? e->row_tags : nullptr;
    fp.filters = filters;
    // the query's bytes in shared memory (the kernel's limit was raised for SA_MAX_DIM at engine creation)
    sa::sa_fixup_kernel<<<2 * e->num_sms, sa::kFixThreads, row_bytes, st>>>(fp);
    SA_CUDA(cudaGetLastError());
    tm.kernels += 1;
    e->scratch_dirty = false;
  }
  SA_CUDA(cudaEventRecord(tm.ev_total[1], st));
  SA_CUDA(cudaEventRecord(e->scratch_free, st));
  // Algorithmic work (DESIGN.md section 5): corpus + inverse norms once per scan launch, queries, results (the rows and
  // queries at their element size; flops are int8 ops for an int8 engine, with the same formula).
  const double n = static_cast<double>(n_rows), d = e->dim, b = nq, es = sa::elem_bytes(e->elem);
  tm.bytes = plan.size() * (n * d * es + n * 4.0) + b * d * es + b * k * 8.0;
  tm.flops = 2.0 * b * n * d;
  e->n_searches += 1;
  return SA_OK;
}

}  // namespace

namespace {
// The epilogue's rule fed chunk by chunk exactly as the kernel feeds it: 32 scores per chunk (the tail chunk padded with
// NaN = masked rows), a shared bound becoming visible at a chunk boundary (the kernel applies it per accumulator).
template <int kKL>
void run_list(const float* score, const int32_t* row, int n, const float* floor_after, float* out_sc, int32_t* out_id,
              float* out_drop) {
  sa::TopList<kKL> L;
  L.init(nullptr);
  float ones[sa::kChunk];
  for (int j = 0; j < sa::kChunk; ++j) ones[j] = 1.0f;
  for (int c0 = 0; c0 < n; c0 += sa::kChunk) {
    float v[sa::kChunk];
    for (int j = 0; j < sa::kChunk; ++j) {
      const int i = c0 + j;
      v[j] = i < n ? score[i] : NAN;
      if (i < n && floor_after && floor_after[i] > -INFINITY) L.apply_shared(sa::float_to_key(floor_after[i]));
    }
    // rows of a chunk are consecutive in the kernel; the hook accepts arbitrary row ids, so the list records positions
    // (c0 + j) and they are translated through row[] at the end
    sa::chunk_process<kKL>(L, v, ones, c0);
  }
  for (int i = 0; i < kKL; ++i) {
    out_sc[i] = L.sc[i];
    out_id[i] = L.id[i] >= 0 ? row[L.id[i]] : -1;
  }
  if (out_drop) *out_drop = L.drop;
}
}  // namespace

extern "C" {

static_assert(sizeof(sa_filter) == sizeof(sa::Filter) && offsetof(sa_filter, all_of) == offsetof(sa::Filter, all_of) &&
                  offsetof(sa_filter, none_of) == offsetof(sa::Filter, none_of) &&
                  offsetof(sa_filter, any_of) == offsetof(sa::Filter, any_of),
              "sa_filter and sa::Filter must share one layout");
static_assert(SA_MAX_K == sa::kDeepMaxK && sa::kFixMaxK >= SA_MAX_K && sa::kShallowMaxK < SA_MAX_K,
              "every k <= SA_MAX_K has a scan variant and fits the fallback's lists");
static_assert(sa::kFixSmemMax == 2 * SA_MAX_DIM, "the fallback's shared memory holds one bf16 query of SA_MAX_DIM");

int sa_version(void) { return 100; }

const char* sa_strerror(int rc) {
  switch (rc) {
    case SA_OK: return "ok";
    case SA_ERR_CUDA: return "CUDA error";
    case SA_ERR_ARG: return "bad argument";
    case SA_ERR_COMM: return "collective error";
    case SA_ERR_CAPACITY: return "capacity exceeded";
    case SA_ERR_DEVICE: return "unsupported device (needs compute capability 9.0 / sm_90a)";
    default: return "unknown status";
  }
}

const char* sa_last_error(void) { return g_err; }

int sa_engine_create(sa_engine** out, int device, int dim, int64_t capacity_rows, int max_batch, int max_k) {
  return sa_engine_create_sim(out, device, dim, capacity_rows, max_batch, max_k, SA_SIM_COSINE);
}

int sa_engine_create_sim(sa_engine** out, int device, int dim, int64_t capacity_rows, int max_batch, int max_k,
                         int similarity) {
  return sa_engine_create_elem(out, device, dim, capacity_rows, max_batch, max_k, similarity, SA_ELEM_BF16);
}

int sa_engine_create_elem(sa_engine** out, int device, int dim, int64_t capacity_rows, int max_batch, int max_k,
                          int similarity, int elem) {
  if (!out) return fail(SA_ERR_ARG, "null out");
  *out = nullptr;
  if (similarity != SA_SIM_COSINE && similarity != SA_SIM_DOT && similarity != SA_SIM_EUCLIDEAN)
    return fail(SA_ERR_ARG, "similarity %d is not SA_SIM_COSINE (0), SA_SIM_DOT (1) or SA_SIM_EUCLIDEAN (2)", similarity);
  if (elem != SA_ELEM_BF16 && elem != SA_ELEM_INT8)
    return fail(SA_ERR_ARG, "elem %d is not SA_ELEM_BF16 (0) or SA_ELEM_INT8 (1)", elem);
  if (dim <= 0 || dim % 64 != 0) return fail(SA_ERR_ARG, "dim %d must be a positive multiple of 64", dim);
  // the fallback scan stages one query row in shared memory; int8: |<q,c>| <= dim 2^14 stays inside int32
  if (dim > SA_MAX_DIM) return fail(SA_ERR_ARG, "dim %d must be at most %d (SA_MAX_DIM)", dim, SA_MAX_DIM);
  // int8: a K slice is 128 elements
  if (elem == SA_ELEM_INT8 && dim % 128 != 0)
    return fail(SA_ERR_ARG, "an int8 index needs dim %d to be a multiple of 128", dim);
  if (capacity_rows <= 0 || capacity_rows >= (1ll << 31) - 512)
    return fail(SA_ERR_ARG, "capacity_rows %lld outside (0, 2^31-512)", (long long)capacity_rows);
  if (max_batch <= 0) return fail(SA_ERR_ARG, "max_batch must be positive");
  if (max_k <= 0 || max_k > SA_MAX_K) return fail(SA_ERR_ARG, "max_k %d outside [1, %d]", max_k, SA_MAX_K);
  int ndev = 0;
  SA_CUDA(cudaGetDeviceCount(&ndev));
  if (device < 0 || device >= ndev) return fail(SA_ERR_ARG, "device %d not present (%d devices)", device, ndev);
  cudaDeviceProp prop;
  SA_CUDA(cudaGetDeviceProperties(&prop, device));
  if (prop.major != 9 || prop.minor != 0)
    return fail(SA_ERR_DEVICE, "device %d is sm_%d%d; this library contains sm_90a code only", device, prop.major,
                prop.minor);
  SA_ON_DEVICE(device);
  if (!get_encode_fn()) return fail(SA_ERR_CUDA, "cuTensorMapEncodeTiled entry point not available");
  // The fallback scan's dynamic shared memory is one query row, 2 SA_MAX_DIM bytes at most: the kernel's limit is set
  // once for that size on this device, so searches of engines with different dims never set it concurrently.
  SA_CUDA(cudaFuncSetAttribute(sa::sa_fixup_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, sa::kFixSmemMax));

  sa_engine* e = new sa_engine();
  e->device = device;
  e->sim = similarity;
  e->elem = elem;
  e->dim = dim;
  e->capacity = capacity_rows;
  e->max_batch = max_batch;
  e->max_k = max_k;
  e->num_sms = prop.multiProcessorCount;
  const size_t part_elems = static_cast<size_t>(e->num_sms) * 128 * 32;
  const size_t qelems = static_cast<size_t>(max_batch) * dim;
  const size_t relems = static_cast<size_t>(max_batch) * max_k;
  e->stage_rows = std::max<int64_t>(1, (64ll << 20) / (static_cast<int64_t>(dim) * 4));
#define SA_TRY(call)                                                                                 \
  do {                                                                                               \
    cudaError_t _e = (call);                                                                         \
    if (_e != cudaSuccess) {                                                                         \
      fail(SA_ERR_CUDA, "%s failed: %s", #call, cudaGetErrorString(_e));                             \
      sa_engine_destroy(e);                                                                          \
      return SA_ERR_CUDA;                                                                            \
    }                                                                                                \
  } while (0)
  SA_TRY(cudaMalloc(&e->part_score, part_elems * sizeof(float)));
  SA_TRY(cudaMalloc(&e->part_idx, part_elems * sizeof(int)));
  SA_TRY(cudaMalloc(&e->part_drop, static_cast<size_t>(e->num_sms) * 128 * sizeof(float)));
  SA_TRY(cudaMalloc(&e->res64, relems * sizeof(double)));
  SA_TRY(cudaMalloc(&e->residx, relems * sizeof(int)));
  SA_TRY(cudaMalloc(&e->fix_entries, static_cast<size_t>(kMaxLaunches) * e->num_sms * 128 * sizeof(sa::FixEntry)));
  SA_TRY(cudaMalloc(&e->fix_query, static_cast<size_t>(max_batch) * sizeof(sa::FixQuery)));
  SA_TRY(cudaMalloc(&e->fix_counters, 2 * sizeof(int)));
  SA_TRY(cudaMalloc(&e->cmax, sizeof(unsigned)));
  SA_TRY(cudaMemset(e->cmax, 0, sizeof(unsigned)));
  SA_TRY(cudaMalloc(&e->prof, static_cast<size_t>(e->num_sms) * sizeof(sa::ScanProf)));
  SA_TRY(cudaMemset(e->prof, 0, static_cast<size_t>(e->num_sms) * sizeof(sa::ScanProf)));
  SA_TRY(cudaMalloc(&e->q_bf16, qelems * 2));
  SA_TRY(cudaMalloc(&e->q_f32, qelems * 4));
  SA_TRY(cudaMalloc(&e->res_score, relems * 4));
  SA_TRY(cudaMalloc(&e->res_idx, relems * 4));
  SA_TRY(cudaMalloc(&e->hits, relems * sizeof(sa::PackedHit)));
  SA_TRY(cudaMalloc(&e->res_row64, relems * sizeof(long long)));
  SA_TRY(cudaMalloc(&e->d_stage, static_cast<size_t>(e->stage_rows) * dim * 4));
  for (int i = 0; i <= kHostSlots; ++i) {
    SA_TRY(cudaHostAlloc(&e->slot[i].h_q, qelems * 4, cudaHostAllocDefault));
    SA_TRY(cudaHostAlloc(&e->slot[i].h_score, relems * 4, cudaHostAllocDefault));
    SA_TRY(cudaHostAlloc(&e->slot[i].h_idx, relems * 4, cudaHostAllocDefault));
    SA_TRY(cudaHostAlloc(&e->slot[i].h_row64, relems * sizeof(long long), cudaHostAllocDefault));
    SA_TRY(cudaHostAlloc(&e->slot[i].h_f, static_cast<size_t>(max_batch) * sizeof(sa::Filter), cudaHostAllocDefault));
    SA_TRY(cudaMalloc(&e->slot[i].d_f, static_cast<size_t>(max_batch) * sizeof(sa::Filter)));
    SA_TRY(cudaEventCreateWithFlags(&e->slot[i].done, cudaEventDisableTiming));
  }
  SA_TRY(cudaHostAlloc(&e->h_stage, static_cast<size_t>(e->stage_rows) * dim * 4, cudaHostAllocDefault));
  // a blocking stream: ordered after work already queued on the legacy default stream (torch's default)
  SA_TRY(cudaStreamCreate(&e->own_stream));
  SA_TRY(cudaEventCreateWithFlags(&e->scratch_free, cudaEventDisableTiming));
  e->thr_n = ((max_batch + 255) / 256) * 256 + 256;
  SA_TRY(cudaMalloc(&e->lane_progress, sizeof(int) * kMaxLaunches * e->num_sms));
  SA_TRY(cudaMalloc(&e->thr_shared, sizeof(unsigned) * e->thr_n));
  SA_TRY(cudaMemset(e->lane_progress, 0, sizeof(int) * kMaxLaunches * e->num_sms));
  SA_TRY(cudaMalloc(&e->lane2, sizeof(unsigned) * kMaxLaunches * e->num_sms * 128));
  SA_TRY(cudaMemset(e->lane2, 0, sizeof(unsigned) * kMaxLaunches * e->num_sms * 128));
  SA_TRY(cudaMemset(e->thr_shared, 0, sizeof(unsigned) * e->thr_n));
  SA_TRY(cudaMemset(e->fix_counters, 0, 2 * sizeof(int)));
  SA_TRY(cudaMemset(e->fix_query, 0, static_cast<size_t>(max_batch) * sizeof(sa::FixQuery)));
  SA_TRY(cudaMalloc(&e->dbg_times, sizeof(long long) * 2 * e->num_sms));
  for (int r = 0; r < kTimingRing; ++r)
    for (int i = 0; i < kMaxLaunches; ++i) e->ring[r].ev_scan[i][0] = e->ring[r].ev_scan[i][1] = nullptr;
  for (int r = 0; r < kTimingRing; ++r) {
    SA_TRY(cudaEventCreate(&e->ring[r].ev_total[0]));
    SA_TRY(cudaEventCreate(&e->ring[r].ev_total[1]));
    for (int i = 0; i < kMaxLaunches; ++i) {
      SA_TRY(cudaEventCreate(&e->ring[r].ev_scan[i][0]));
      SA_TRY(cudaEventCreate(&e->ring[r].ev_scan[i][1]));
    }
  }
#undef SA_TRY
  *out = e;
  return SA_OK;
}

void sa_engine_destroy(sa_engine* e) {
  if (!e) return;
  DeviceGuard dg(e->device);  // the caller's current device is restored on return
  cudaDeviceSynchronize();
  cudaFree(e->part_score);
  cudaFree(e->part_idx);
  cudaFree(e->part_drop);
  cudaFree(e->res64);
  cudaFree(e->residx);
  cudaFree(e->fix_entries);
  cudaFree(e->fix_query);
  cudaFree(e->fix_counters);
  cudaFree(e->cmax);
  cudaFree(e->prof);
  cudaFree(e->q_bf16);
  cudaFree(e->q_f32);
  cudaFree(e->res_score);
  cudaFree(e->res_idx);
  cudaFree(e->hits);
  cudaFree(e->res_row64);
  cudaFree(e->d_stage);
  for (int i = 0; i <= kHostSlots; ++i) {
    cudaFreeHost(e->slot[i].h_q);
    cudaFreeHost(e->slot[i].h_score);
    cudaFreeHost(e->slot[i].h_idx);
    cudaFreeHost(e->slot[i].h_row64);
    cudaFreeHost(e->slot[i].h_f);
    cudaFree(e->slot[i].d_f);
    if (e->slot[i].done) cudaEventDestroy(e->slot[i].done);
  }
  cudaFreeHost(e->h_stage);
  if (e->own_stream) cudaStreamDestroy(e->own_stream);
  if (e->scratch_free) cudaEventDestroy(e->scratch_free);
  cudaFree(e->lane_progress);
  cudaFree(e->lane2);
  cudaFree(e->thr_shared);
  cudaFree(e->dbg_times);
  for (int r = 0; r < kTimingRing; ++r) {
    for (int i = 0; i < 2; ++i)
      if (e->ring[r].ev_total[i]) cudaEventDestroy(e->ring[r].ev_total[i]);
    for (int i = 0; i < kMaxLaunches; ++i)
      for (int j = 0; j < 2; ++j)
        if (e->ring[r].ev_scan[i][j]) cudaEventDestroy(e->ring[r].ev_scan[i][j]);
  }
  delete e;
}

namespace {
constexpr int kIngestBlock = 256;  // one warp per row
unsigned ingest_grid(int64_t n) { return static_cast<unsigned>((n * 32 + kIngestBlock - 1) / kIngestBlock); }
}  // namespace

int sa_corpus_bind(sa_engine* e, void* rows_dev, float* row_term_dev, int64_t n_valid) {
  if (!e || !rows_dev || !row_term_dev) return fail(SA_ERR_ARG, "null argument");
  if (reinterpret_cast<uintptr_t>(rows_dev) % 16) return fail(SA_ERR_ARG, "corpus must be 16-byte aligned");
  if (reinterpret_cast<uintptr_t>(row_term_dev) % 16) return fail(SA_ERR_ARG, "row_term must be 16-byte aligned");
  if (n_valid < 0 || n_valid > e->capacity) return fail(SA_ERR_CAPACITY, "n_valid outside [0, capacity]");
  SA_ON_DEVICE(e->device);
  int rc = encode_rows_map(&e->tmap_c[0], rows_dev, static_cast<uint64_t>(e->capacity), e->dim,
                           sa::ScanCfg<1>::kBRows, e->elem);
  if (rc) return rc;
  rc = encode_rows_map(&e->tmap_c[1], rows_dev, static_cast<uint64_t>(e->capacity), e->dim,
                       sa::ScanCfg<2>::kBRows, e->elem);
  if (rc) return rc;
  e->corpus = rows_dev;
  e->row_term = row_term_dev;
  e->n_rows = n_valid;
  e->bound = true;
  if (e->sim != SA_SIM_COSINE) {
    // Cmax over the rows taken as committed (the legacy default stream orders this before later work on blocking streams)
    SA_CUDA(cudaMemsetAsync(e->cmax, 0, sizeof(unsigned), 0));
    if (n_valid > 0) {
      if (e->elem == SA_ELEM_INT8)
        sa::sa_rowterm_i8_kernel<<<ingest_grid(n_valid), kIngestBlock, 0, 0>>>(static_cast<const int8_t*>(e->corpus),
                                                                              nullptr, -1, n_valid, e->dim, e->sim, e->cmax);
      else
        sa::sa_rowterm_kernel<sa::kSimDot><<<ingest_grid(n_valid), kIngestBlock, 0, 0>>>(
            static_cast<const uint16_t*>(e->corpus), nullptr, -1, n_valid, e->dim, e->cmax);
      SA_CUDA(cudaGetLastError());
    }
  }
  return SA_OK;
}

int sa_corpus_bind_tags(sa_engine* e, uint64_t* row_tags_dev) {
  if (!e) return fail(SA_ERR_ARG, "null engine");
  if (reinterpret_cast<uintptr_t>(row_tags_dev) % 16) return fail(SA_ERR_ARG, "row tags must be 16-byte aligned");
  e->row_tags = reinterpret_cast<unsigned long long*>(row_tags_dev);
  return SA_OK;
}

int sa_corpus_commit(sa_engine* e, int64_t first_row, int64_t n_new, uintptr_t stream) {
  int rc = check_engine(e);
  if (rc) return rc;
  if (first_row != e->n_rows) return fail(SA_ERR_ARG, "commit must start at the current row count %lld", (long long)e->n_rows);
  if (n_new < 0 || first_row + n_new > e->capacity) return fail(SA_ERR_CAPACITY, "commit past capacity");
  if (n_new == 0) return SA_OK;
  SA_ON_DEVICE(e->device);
  const cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const uint16_t* rows = static_cast<const uint16_t*>(e->corpus);
  if (e->elem == SA_ELEM_INT8)
    sa::sa_rowterm_i8_kernel<<<ingest_grid(n_new), kIngestBlock, 0, st>>>(static_cast<const int8_t*>(e->corpus),
                                                                         e->row_term, first_row, n_new, e->dim, e->sim,
                                                                         e->cmax);
  else if (e->sim == SA_SIM_COSINE)
    sa::sa_rownorm_kernel<<<ingest_grid(n_new), kIngestBlock, 0, st>>>(rows, e->row_term, first_row, n_new, e->dim);
  else if (e->sim == SA_SIM_DOT)
    sa::sa_rowterm_kernel<sa::kSimDot><<<ingest_grid(n_new), kIngestBlock, 0, st>>>(rows, e->row_term, first_row,
                                                                                   n_new, e->dim, e->cmax);
  else
    sa::sa_rowterm_kernel<sa::kSimEuc><<<ingest_grid(n_new), kIngestBlock, 0, st>>>(rows, e->row_term, first_row,
                                                                                   n_new, e->dim, e->cmax);
  SA_CUDA(cudaGetLastError());
  e->n_rows = first_row + n_new;
  return SA_OK;
}

int sa_corpus_append_f32(sa_engine* e, const float* rows_f32_dev, int64_t n_new, uintptr_t stream) {
  int rc = check_engine(e);
  if (rc) return rc;
  if (!rows_f32_dev) return fail(SA_ERR_ARG, "null rows");
  if (n_new < 0 || e->n_rows + n_new > e->capacity) return fail(SA_ERR_CAPACITY, "append past capacity");
  if (n_new == 0) return SA_OK;
  SA_ON_DEVICE(e->device);
  const cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  float* w = e->row_term + e->n_rows;
  uint16_t* dst = static_cast<uint16_t*>(e->corpus) + e->n_rows * e->dim;
  if (e->elem == SA_ELEM_INT8)
    sa::sa_convert_rows_i8_kernel<<<ingest_grid(n_new), kIngestBlock, 0, st>>>(
        rows_f32_dev, static_cast<int8_t*>(e->corpus) + e->n_rows * e->dim, w, n_new, e->dim, e->sim, e->cmax);
  else if (e->sim == SA_SIM_COSINE)
    sa::sa_convert_rows_kernel<<<ingest_grid(n_new), kIngestBlock, 0, st>>>(rows_f32_dev, dst, w, n_new, e->dim);
  else if (e->sim == SA_SIM_DOT)
    sa::sa_convert_rows_term_kernel<sa::kSimDot><<<ingest_grid(n_new), kIngestBlock, 0, st>>>(rows_f32_dev, dst, w, n_new,
                                                                                            e->dim, e->cmax);
  else
    sa::sa_convert_rows_term_kernel<sa::kSimEuc><<<ingest_grid(n_new), kIngestBlock, 0, st>>>(rows_f32_dev, dst, w, n_new,
                                                                                            e->dim, e->cmax);
  SA_CUDA(cudaGetLastError());
  e->n_rows += n_new;
  return SA_OK;
}

int sa_corpus_append_host_f32(sa_engine* e, const float* rows_f32_host, int64_t n_new) {
  int rc = check_engine(e);
  if (rc) return rc;
  if (!rows_f32_host) return fail(SA_ERR_ARG, "null rows");
  if (n_new < 0 || e->n_rows + n_new > e->capacity) return fail(SA_ERR_CAPACITY, "append past capacity");
  SA_ON_DEVICE(e->device);
  int64_t done = 0;
  while (done < n_new) {
    const int64_t n = std::min(e->stage_rows, n_new - done);
    const size_t bytes = static_cast<size_t>(n) * e->dim * 4;
    memcpy(e->h_stage, rows_f32_host + done * e->dim, bytes);
    SA_CUDA(cudaMemcpyAsync(e->d_stage, e->h_stage, bytes, cudaMemcpyHostToDevice, e->own_stream));
    rc = sa_corpus_append_f32(e, e->d_stage, n, reinterpret_cast<uintptr_t>(e->own_stream));
    if (rc) return rc;
    SA_CUDA(cudaStreamSynchronize(e->own_stream));  // staging buffers are reused by the next chunk
    done += n;
  }
  return SA_OK;
}

int sa_corpus_reset(sa_engine* e) {
  if (!e) return fail(SA_ERR_ARG, "null engine");
  if (e->sim != SA_SIM_COSINE) {
    // Cmax starts over.  Blocking: an append issued after the reset, on any stream, must raise it after it was cleared.
    SA_ON_DEVICE(e->device);
    SA_CUDA(cudaDeviceSynchronize());
    SA_CUDA(cudaMemset(e->cmax, 0, sizeof(unsigned)));
    SA_CUDA(cudaDeviceSynchronize());
  }
  e->n_rows = 0;
  return SA_OK;
}

int64_t sa_corpus_rows(const sa_engine* e) { return e ? e->n_rows : -1; }

int sa_search(sa_engine* e, const void* q_bf16_dev, int nq, int k, float* out_score_dev, int32_t* out_idx_dev,
              double* out_score64_dev, uintptr_t stream) {
  int rc = check_engine(e);
  if (rc) return rc;
  return do_search(e, q_bf16_dev, nq, k, out_score_dev, out_idx_dev, out_score64_dev,
                   nullptr, 0, reinterpret_cast<cudaStream_t>(stream));
}

int sa_search_filtered(sa_engine* e, const void* q_bf16_dev, const sa_filter* filters_dev, int nq, int k,
                       float* out_score_dev, int32_t* out_idx_dev, double* out_score64_dev, uintptr_t stream) {
  int rc = check_search(e, filters_dev, true);
  if (rc) return rc;
  return do_search(e, q_bf16_dev, nq, k, out_score_dev, out_idx_dev, out_score64_dev,
                   nullptr, 0, reinterpret_cast<cudaStream_t>(stream), reinterpret_cast<const sa::Filter*>(filters_dev));
}

static int search_f32(sa_engine* e, const float* q_f32_dev, const sa_filter* filters_dev, bool filtered, int nq, int k,
                      float* out_score_dev, int32_t* out_idx_dev, double* out_score64_dev, uintptr_t stream) {
  int rc = check_search(e, filters_dev, filtered);
  if (rc) return rc;
  if (!q_f32_dev) return fail(SA_ERR_ARG, "null queries");
  if (nq <= 0 || nq > e->max_batch) return fail(SA_ERR_CAPACITY, "nq %d outside [1, max_batch %d]", nq, e->max_batch);
  SA_ON_DEVICE(e->device);
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  rc = convert_queries(e, q_f32_dev, nq, st);
  if (rc) return rc;
  rc = do_search(e, e->q_bf16, nq, k, out_score_dev, out_idx_dev, out_score64_dev, nullptr, 0, st,
                 reinterpret_cast<const sa::Filter*>(filters_dev));
  if (rc == SA_OK) e->ring[(e->n_searches - 1) % kTimingRing].kernels += 1;
  return rc;
}

int sa_search_f32(sa_engine* e, const float* q_f32_dev, int nq, int k, float* out_score_dev, int32_t* out_idx_dev,
                  double* out_score64_dev, uintptr_t stream) {
  return search_f32(e, q_f32_dev, nullptr, false, nq, k, out_score_dev, out_idx_dev, out_score64_dev, stream);
}

int sa_search_f32_filtered(sa_engine* e, const float* q_f32_dev, const sa_filter* filters_dev, int nq, int k,
                           float* out_score_dev, int32_t* out_idx_dev, double* out_score64_dev, uintptr_t stream) {
  return search_f32(e, q_f32_dev, filters_dev, true, nq, k, out_score_dev, out_idx_dev, out_score64_dev, stream);
}

namespace {
// ------------------------------------------------------------------------------------------------------------------
// Multi-GPU exchange (SURVEY.md section 8e): every rank scans its row shard, ONE all-gather of the packed per-query
// (cosine f64, global row) lists -- nq*k*16 bytes per rank -- and a k-way merge on every rank.  NCCL is loaded at run
// time: the copy already in the process if there is one (torch's), else SA_NCCL_LIB / sa_comm_set_library, else the
// system libnccl.so.2 -- so exactly one NCCL ever lives in the process.
// ------------------------------------------------------------------------------------------------------------------
struct NcclApi {
  void* handle = nullptr;
  ncclResult_t (*GetVersion)(int*) = nullptr;
  ncclResult_t (*GetUniqueId)(ncclUniqueId*) = nullptr;
  ncclResult_t (*CommInitRank)(ncclComm_t*, int, ncclUniqueId, int) = nullptr;
  ncclResult_t (*CommInitAll)(ncclComm_t*, int, const int*) = nullptr;
  ncclResult_t (*CommDestroy)(ncclComm_t) = nullptr;
  ncclResult_t (*AllGather)(const void*, void*, size_t, ncclDataType_t, ncclComm_t, cudaStream_t) = nullptr;
  ncclResult_t (*GroupStart)() = nullptr;
  ncclResult_t (*GroupEnd)() = nullptr;
  const char* (*GetErrorString)(ncclResult_t) = nullptr;
  std::string path;
};
NcclApi g_nccl;
std::string g_nccl_path_hint;

int load_nccl() {
  if (g_nccl.handle) return SA_OK;
  std::vector<std::string> tried;
  void* h = dlopen("libnccl.so.2", RTLD_NOW | RTLD_NOLOAD);  // already in the process (torch imported)?
  std::string from = "already loaded libnccl.so.2";
  auto try_path = [&](const std::string& pth) {
    if (h || pth.empty()) return;
    h = dlopen(pth.c_str(), RTLD_NOW | RTLD_GLOBAL);
    if (h) from = pth;
    else tried.push_back(pth);
  };
  try_path(g_nccl_path_hint);
  if (const char* env = getenv("SA_NCCL_LIB")) try_path(env);
  try_path("libnccl.so.2");
  try_path("libnccl.so");
  if (!h) {
    std::string msg;
    for (auto& t : tried) msg += " " + t;
    return fail(SA_ERR_COMM, "NCCL not found (tried:%s); set SA_NCCL_LIB or call sa_comm_set_library", msg.c_str());
  }
#define SA_NCCL_SYM(field, name)                                                          \
  g_nccl.field = reinterpret_cast<decltype(g_nccl.field)>(dlsym(h, name));                \
  if (!g_nccl.field) return fail(SA_ERR_COMM, "%s lacks symbol %s", from.c_str(), name)
  SA_NCCL_SYM(GetVersion, "ncclGetVersion");
  SA_NCCL_SYM(GetUniqueId, "ncclGetUniqueId");
  SA_NCCL_SYM(CommInitRank, "ncclCommInitRank");
  SA_NCCL_SYM(CommInitAll, "ncclCommInitAll");
  SA_NCCL_SYM(CommDestroy, "ncclCommDestroy");
  SA_NCCL_SYM(AllGather, "ncclAllGather");
  SA_NCCL_SYM(GroupStart, "ncclGroupStart");
  SA_NCCL_SYM(GroupEnd, "ncclGroupEnd");
  SA_NCCL_SYM(GetErrorString, "ncclGetErrorString");
#undef SA_NCCL_SYM
  g_nccl.handle = h;
  g_nccl.path = from;
  return SA_OK;
}

#define SA_NCCL(call)                                                                                          \
  do {                                                                                                         \
    ncclResult_t _r = (call);                                                                                  \
    if (_r != ncclSuccess)                                                                                     \
      return fail(SA_ERR_COMM, "%s failed: %s (%s:%d)", #call, g_nccl.GetErrorString(_r), __FILE__, __LINE__); \
  } while (0)

}  // namespace

struct sa_comm {
  int n_ranks = 0;
  int rank = -1;                    // >= 0: one rank of a multi-process communicator; -1: single process, all ranks here
  std::vector<int> devices;         // device of each local rank
  std::vector<ncclComm_t> comms;    // one per local rank
  std::vector<sa::PackedHit*> gathered;  // per local rank: [n_ranks][cap_nq][cap_k], grown on demand
  std::vector<size_t> gathered_elems;
  int sim = -1;                     // one process per GPU: the similarity every rank's engine was found to have ...
  int elem = -1;                    // ... and its element type
};

namespace {

int comm_gather_buffer(sa_comm* c, int local, int nq, int k, sa::PackedHit** out) {
  const size_t need = static_cast<size_t>(c->n_ranks) * nq * k;
  if (c->gathered_elems[local] < need) {
    DeviceGuard g(c->devices[local]);
    if (c->gathered[local]) {
      cudaDeviceSynchronize();  // growth is rare (first call, or a larger batch than ever before)
      cudaFree(c->gathered[local]);
      c->gathered[local] = nullptr;
      c->gathered_elems[local] = 0;
    }
    SA_CUDA(cudaMalloc(&c->gathered[local], need * sizeof(sa::PackedHit)));
    c->gathered_elems[local] = need;
  }
  *out = c->gathered[local];
  return SA_OK;
}

// This rank's part of a sharded search on stream st: shard scan -> packed hits -> all-gather -> merge.  `phases` selects
// the steps (bit 0 scan, bit 1 all-gather, bit 2 merge) so a single process driving several GPUs can put the collectives
// of all its ranks into one NCCL group (inside a group the collective is only enqueued at ncclGroupEnd, so nothing that
// must follow it on the stream may be issued before the group closes).
int sharded_search_on_stream(sa_comm* c, int local, sa_engine* e, const void* q_dev, int nq, int k,
                             int64_t row_offset, float* out_score_dev, long long* out_row_dev, cudaStream_t st,
                             int phases = 7, const sa::Filter* filters = nullptr) {
  int rc;
  if (phases & 1) {
    rc = do_search(e, q_dev, nq, k, e->res_score, e->res_idx, nullptr, e->hits, row_offset, st, filters);
    if (rc) return rc;
  }
  sa::PackedHit* gathered = nullptr;
  rc = comm_gather_buffer(c, local, nq, k, &gathered);
  if (rc) return rc;
  if (phases & 2) {
    const size_t bytes = static_cast<size_t>(nq) * k * sizeof(sa::PackedHit);
    SA_NCCL(g_nccl.AllGather(e->hits, gathered, bytes, ncclChar, c->comms[local], st));
  }
  if (phases & 4) {
    rc = launch_merge_packed(gathered, c->n_ranks, nq, k, out_score_dev, out_row_dev, e->sim == SA_SIM_EUCLIDEAN, st);
    if (rc) return rc;
    e->ring[(e->n_searches - 1) % kTimingRing].kernels += 2;  // the collective and the shard merge
  }
  return SA_OK;
}

// Host-buffer search into slot si.  comm == nullptr: this engine alone (shard-local int32 rows); otherwise this rank's
// part of a sharded search (global int64 rows, identical on every rank).  `phases` as in sharded_search_on_stream
// (bit 0 also covers the H2D copy and the conversion, bit 2 the D2H copies and the slot's event).  filters_host ([nq],
// or nullptr: unfiltered) is staged through the slot's pinned buffer, so it may be reused as soon as submit returns.
int host_submit(sa_engine* e, int si, const float* q_f32_host, int nq, int k, sa_comm* c, int local, int64_t row_offset,
                int phases = 7, const sa_filter* filters_host = nullptr) {
  sa_engine::HostSlot& sl = e->slot[si];
  SA_ON_DEVICE(e->device);
  cudaStream_t st = e->own_stream;
  const size_t rbytes = static_cast<size_t>(nq) * k * 4;
  if (phases & 1) {
    if (sl.busy) return fail(SA_ERR_ARG, "host slot %d still holds an unwaited search", si);
    if (!q_f32_host) return fail(SA_ERR_ARG, "null buffer");
    if (nq <= 0 || nq > e->max_batch) return fail(SA_ERR_CAPACITY, "nq %d outside [1, max_batch %d]", nq, e->max_batch);
    if (k <= 0 || k > e->max_k) return fail(SA_ERR_ARG, "k %d outside [1, max_k %d]", k, e->max_k);
    const size_t qbytes = static_cast<size_t>(nq) * e->dim * 4;
    // A query buffer that is already page-locked (sa_host_alloc, cudaHostRegister, torch pin_memory) is DMA'd
    // directly -- the caller then keeps it unchanged until the matching wait; pageable memory is staged.
    const float* q_src = q_f32_host;
    if (!is_pinned(q_f32_host)) {
      memcpy(sl.h_q, q_f32_host, qbytes);
      q_src = sl.h_q;
    }
    SA_CUDA(cudaMemcpyAsync(e->q_f32, q_src, qbytes, cudaMemcpyHostToDevice, st));
    if (filters_host != nullptr) {
      // the slot's device copy is read until the search's last kernel; the slot is not reused before its wait
      memcpy(sl.h_f, filters_host, static_cast<size_t>(nq) * sizeof(sa::Filter));
      SA_CUDA(cudaMemcpyAsync(sl.d_f, sl.h_f, static_cast<size_t>(nq) * sizeof(sa::Filter), cudaMemcpyHostToDevice, st));
    }
    int rc = convert_queries(e, e->q_f32, nq, st);
    if (rc) return rc;
    if (c == nullptr) {
      rc = do_search(e, e->q_bf16, nq, k, e->res_score, e->res_idx, nullptr, nullptr, 0, st,
                     filters_host != nullptr ? sl.d_f : nullptr);
      if (rc) return rc;
    }
  }
  if (c != nullptr) {
    int rc = sharded_search_on_stream(c, local, e, e->q_bf16, nq, k, row_offset, e->res_score, e->res_row64, st, phases,
                                      filters_host != nullptr ? sl.d_f : nullptr);
    if (rc) return rc;
  }
  if (phases & 4) {
    SA_CUDA(cudaMemcpyAsync(sl.h_score, e->res_score, rbytes, cudaMemcpyDeviceToHost, st));
    if (c == nullptr) SA_CUDA(cudaMemcpyAsync(sl.h_idx, e->res_idx, rbytes, cudaMemcpyDeviceToHost, st));
    else SA_CUDA(cudaMemcpyAsync(sl.h_row64, e->res_row64, 2 * rbytes, cudaMemcpyDeviceToHost, st));
    e->ring[(e->n_searches - 1) % kTimingRing].kernels += 1;  // the fp32 -> bf16 conversion
    SA_CUDA(cudaEventRecord(sl.done, st));
    sl.nq = nq;
    sl.k = k;
    sl.sharded = c != nullptr;
    sl.busy = true;
  }
  return SA_OK;
}

int host_wait(sa_engine* e, int si, float* out_score_host, void* out_idx_host, bool sharded) {
  sa_engine::HostSlot& sl = e->slot[si];
  if (!sl.busy) return fail(SA_ERR_ARG, "host slot %d has no search in flight", si);
  if (sl.sharded != sharded) return fail(SA_ERR_ARG, "host slot %d holds a %s search", si, sl.sharded ? "sharded" : "local");
  if (!out_score_host || !out_idx_host) return fail(SA_ERR_ARG, "null buffer");
  SA_ON_DEVICE(e->device);
  SA_CUDA(cudaEventSynchronize(sl.done));
  const size_t rbytes = static_cast<size_t>(sl.nq) * sl.k * 4;
  memcpy(out_score_host, sl.h_score, rbytes);
  if (sharded) memcpy(out_idx_host, sl.h_row64, 2 * rbytes);
  else memcpy(out_idx_host, sl.h_idx, rbytes);
  sl.busy = false;
  return SA_OK;
}

}  // namespace

static int search_host(sa_engine* e, const float* q_f32_host, const sa_filter* filters_host, bool filtered, int nq,
                       int k, float* out_score_host, int32_t* out_idx_host) {
  int rc = check_search(e, filters_host, filtered);
  if (rc) return rc;
  if (!out_score_host || !out_idx_host) return fail(SA_ERR_ARG, "null buffer");
  e->slot[kHostSlots].busy = false;  // the private slot of the blocking call
  rc = host_submit(e, kHostSlots, q_f32_host, nq, k, nullptr, 0, 0, 7, filters_host);
  if (rc) return rc;
  return host_wait(e, kHostSlots, out_score_host, out_idx_host, false);
}

int sa_search_host(sa_engine* e, const float* q_f32_host, int nq, int k, float* out_score_host,
                   int32_t* out_idx_host) {
  return search_host(e, q_f32_host, nullptr, false, nq, k, out_score_host, out_idx_host);
}

int sa_search_host_filtered(sa_engine* e, const float* q_f32_host, const sa_filter* filters_host, int nq, int k,
                            float* out_score_host, int32_t* out_idx_host) {
  return search_host(e, q_f32_host, filters_host, true, nq, k, out_score_host, out_idx_host);
}

static int search_host_submit(sa_engine* e, int slot, const float* q_f32_host, const sa_filter* filters_host,
                              bool filtered, int nq, int k) {
  int rc = check_search(e, filters_host, filtered);
  if (rc) return rc;
  if (slot < 0 || slot >= kHostSlots) return fail(SA_ERR_ARG, "slot %d outside [0, %d)", slot, kHostSlots);
  return host_submit(e, slot, q_f32_host, nq, k, nullptr, 0, 0, 7, filters_host);
}

int sa_search_host_submit(sa_engine* e, int slot, const float* q_f32_host, int nq, int k) {
  return search_host_submit(e, slot, q_f32_host, nullptr, false, nq, k);
}

int sa_search_host_submit_filtered(sa_engine* e, int slot, const float* q_f32_host, const sa_filter* filters_host, int nq,
                                   int k) {
  return search_host_submit(e, slot, q_f32_host, filters_host, true, nq, k);
}

int sa_search_host_wait(sa_engine* e, int slot, float* out_score_host, int32_t* out_idx_host) {
  int rc = check_engine(e);
  if (rc) return rc;
  if (slot < 0 || slot >= kHostSlots) return fail(SA_ERR_ARG, "slot %d outside [0, %d)", slot, kHostSlots);
  return host_wait(e, slot, out_score_host, out_idx_host, false);
}

int sa_merge_shards(sa_engine* e, const double* score64_dev, const int64_t* global_idx_dev, int n_shards, int nq,
                    int k, float* out_score_dev, int64_t* out_idx_dev, uintptr_t stream) {
  if (!e || !score64_dev || !global_idx_dev || !out_score_dev || !out_idx_dev) return fail(SA_ERR_ARG, "null argument");
  if (n_shards <= 0 || n_shards > 64) return fail(SA_ERR_ARG, "n_shards %d outside [1, 64]", n_shards);
  if (nq <= 0 || k <= 0) return fail(SA_ERR_ARG, "nq and k must be positive");
  SA_ON_DEVICE(e->device);
  sa::sa_merge_serial_kernel<<<(nq + 127) / 128, 128, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      sa::SplitHits{score64_dev, reinterpret_cast<const long long*>(global_idx_dev)}, n_shards, nq, k, out_score_dev,
      reinterpret_cast<long long*>(out_idx_dev), e->sim == SA_SIM_EUCLIDEAN);
  SA_CUDA(cudaGetLastError());
  return SA_OK;
}

static int search_hits(sa_engine* e, const void* q_bf16_dev, const sa_filter* filters_dev, bool filtered, int nq, int k,
                       int64_t row_offset, sa_hit* out_hits_dev, uintptr_t stream) {
  int rc = check_search(e, filters_dev, filtered);
  if (rc) return rc;
  if (!out_hits_dev) return fail(SA_ERR_ARG, "null buffer");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  {
    SA_ON_DEVICE(e->device);
    SA_CUDA(cudaStreamWaitEvent(st, e->scratch_free, 0));  // res_score / res_idx below are engine scratch
  }
  return do_search(e, q_bf16_dev, nq, k, e->res_score, e->res_idx, nullptr,
                   reinterpret_cast<sa::PackedHit*>(out_hits_dev), row_offset, st,
                   reinterpret_cast<const sa::Filter*>(filters_dev));
}

int sa_search_hits(sa_engine* e, const void* q_bf16_dev, int nq, int k, int64_t row_offset, sa_hit* out_hits_dev,
                   uintptr_t stream) {
  return search_hits(e, q_bf16_dev, nullptr, false, nq, k, row_offset, out_hits_dev, stream);
}

int sa_search_hits_filtered(sa_engine* e, const void* q_bf16_dev, const sa_filter* filters_dev, int nq, int k,
                            int64_t row_offset, sa_hit* out_hits_dev, uintptr_t stream) {
  return search_hits(e, q_bf16_dev, filters_dev, true, nq, k, row_offset, out_hits_dev, stream);
}

int sa_merge_hits(sa_engine* e, const sa_hit* hits_dev, int n_shards, int nq, int k, float* out_score_dev,
                  int64_t* out_row_dev, uintptr_t stream) {
  if (!e || !hits_dev || !out_score_dev || !out_row_dev) return fail(SA_ERR_ARG, "null argument");
  if (n_shards <= 0 || n_shards > 64) return fail(SA_ERR_ARG, "n_shards %d outside [1, 64]", n_shards);
  if (nq <= 0 || k <= 0) return fail(SA_ERR_ARG, "nq and k must be positive");
  SA_ON_DEVICE(e->device);
  return launch_merge_packed(reinterpret_cast<const sa::PackedHit*>(hits_dev), n_shards, nq, k, out_score_dev,
                             reinterpret_cast<long long*>(out_row_dev), e->sim == SA_SIM_EUCLIDEAN,
                             reinterpret_cast<cudaStream_t>(stream));
}

// ---- communicator ---------------------------------------------------------------------------------------------------
int sa_comm_set_library(const char* path) {
  g_nccl_path_hint = path ? path : "";
  return SA_OK;
}

int sa_comm_nccl_version(int* version, char* path_out, int path_cap) {
  int rc = load_nccl();
  if (rc) return rc;
  if (version) SA_NCCL(g_nccl.GetVersion(version));
  if (path_out && path_cap > 0) snprintf(path_out, path_cap, "%s", g_nccl.path.c_str());
  return SA_OK;
}

int sa_comm_unique_id(void* id_out_128) {
  if (!id_out_128) return fail(SA_ERR_ARG, "null id");
  int rc = load_nccl();
  if (rc) return rc;
  static_assert(sizeof(ncclUniqueId) == SA_COMM_ID_BYTES, "SA_COMM_ID_BYTES must match ncclUniqueId");
  ncclUniqueId id;
  SA_NCCL(g_nccl.GetUniqueId(&id));
  memcpy(id_out_128, &id, sizeof id);
  return SA_OK;
}

int sa_comm_create_rank(sa_comm** out, int n_ranks, int rank, const void* id_128, int device) {
  if (!out || !id_128) return fail(SA_ERR_ARG, "null argument");
  *out = nullptr;
  if (n_ranks <= 0 || n_ranks > 64 || rank < 0 || rank >= n_ranks) return fail(SA_ERR_ARG, "bad rank %d of %d", rank, n_ranks);
  int rc = load_nccl();
  if (rc) return rc;
  SA_ON_DEVICE(device);
  ncclUniqueId id;
  memcpy(&id, id_128, sizeof id);
  ncclComm_t comm = nullptr;
  SA_NCCL(g_nccl.CommInitRank(&comm, n_ranks, id, rank));
  sa_comm* c = new sa_comm();
  c->n_ranks = n_ranks;
  c->rank = rank;
  c->devices.push_back(device);
  c->comms.push_back(comm);
  c->gathered.push_back(nullptr);
  c->gathered_elems.push_back(0);
  *out = c;
  return SA_OK;
}

int sa_comm_create(sa_comm** out, int n_gpus, const int* devices) {
  if (!out) return fail(SA_ERR_ARG, "null out");
  *out = nullptr;
  if (n_gpus <= 0 || n_gpus > 64) return fail(SA_ERR_ARG, "n_gpus %d outside [1, 64]", n_gpus);
  int rc = load_nccl();
  if (rc) return rc;
  sa_comm* c = new sa_comm();
  c->n_ranks = n_gpus;
  c->rank = -1;
  for (int g = 0; g < n_gpus; ++g) c->devices.push_back(devices ? devices[g] : g);
  c->comms.assign(n_gpus, nullptr);
  c->gathered.assign(n_gpus, nullptr);
  c->gathered_elems.assign(n_gpus, 0);
  int prev = 0;
  cudaGetDevice(&prev);
  ncclResult_t r = g_nccl.CommInitAll(c->comms.data(), n_gpus, c->devices.data());
  cudaSetDevice(prev);
  if (r != ncclSuccess) {
    delete c;
    return fail(SA_ERR_COMM, "ncclCommInitAll failed: %s", g_nccl.GetErrorString(r));
  }
  *out = c;
  return SA_OK;
}

void sa_comm_destroy(sa_comm* c) {
  if (!c) return;
  for (size_t i = 0; i < c->comms.size(); ++i) {
    DeviceGuard g(c->devices[i]);
    cudaDeviceSynchronize();
    if (c->gathered[i]) cudaFree(c->gathered[i]);
    if (c->comms[i] && g_nccl.CommDestroy) g_nccl.CommDestroy(c->comms[i]);
  }
  delete c;
}

int sa_comm_ranks(const sa_comm* c) { return c ? c->n_ranks : -1; }

namespace {
int check_rank_comm(sa_comm* c, const sa_engine* e) {
  if (!c) return fail(SA_ERR_ARG, "null communicator");
  if (c->rank < 0) return fail(SA_ERR_ARG, "single-process communicator: use sa_gather_merge");
  if (c->devices[0] != e->device) return fail(SA_ERR_ARG, "communicator is on device %d, engine on %d", c->devices[0], e->device);
  if (c->sim >= 0) {
    if (c->sim != e->sim) return fail(SA_ERR_ARG, "engine has similarity %d, the communicator's ranks %d", e->sim, c->sim);
    if (c->elem != e->elem)
      return fail(SA_ERR_ARG, "engine has element type %d, the communicator's ranks %d", e->elem, c->elem);
    return SA_OK;
  }
  // First search on this communicator (a collective, like the search itself): all-gather every rank's (similarity,
  // element type) once; shards ranked under different similarities, or holding other element types, cannot be merged.
  SA_ON_DEVICE(e->device);
  int* d = nullptr;
  SA_CUDA(cudaMalloc(&d, sizeof(int) * 2 * (c->n_ranks + 1)));
  std::vector<int> got(2 * c->n_ranks, -1);
  const int mine[2] = {e->sim, e->elem};
  cudaError_t ce = cudaMemcpy(d + 2 * c->n_ranks, mine, sizeof mine, cudaMemcpyHostToDevice);
  ncclResult_t nr = ncclSuccess;
  if (ce == cudaSuccess) nr = g_nccl.AllGather(d + 2 * c->n_ranks, d, 2, ncclInt32, c->comms[0], e->own_stream);
  if (ce == cudaSuccess && nr == ncclSuccess) ce = cudaStreamSynchronize(e->own_stream);
  if (ce == cudaSuccess && nr == ncclSuccess)
    ce = cudaMemcpy(got.data(), d, sizeof(int) * 2 * c->n_ranks, cudaMemcpyDeviceToHost);
  cudaFree(d);
  if (nr != ncclSuccess) return fail(SA_ERR_COMM, "similarity all-gather failed: %s", g_nccl.GetErrorString(nr));
  if (ce != cudaSuccess) return fail(SA_ERR_CUDA, "similarity all-gather: %s", cudaGetErrorString(ce));
  for (int r = 0; r < c->n_ranks; ++r) {
    if (got[2 * r] != e->sim) return fail(SA_ERR_ARG, "rank %d has similarity %d, this rank %d", r, got[2 * r], e->sim);
    if (got[2 * r + 1] != e->elem)
      return fail(SA_ERR_ARG, "rank %d has element type %d, this rank %d", r, got[2 * r + 1], e->elem);
  }
  c->sim = e->sim;
  c->elem = e->elem;
  return SA_OK;
}
}  // namespace

static int sharded_search(sa_comm* c, sa_engine* e, const void* q_bf16_dev, const sa_filter* filters_dev, bool filtered,
                          int nq, int k, int64_t row_offset, float* out_score_dev, int64_t* out_row_dev,
                          uintptr_t stream) {
  int rc = check_search(e, filters_dev, filtered);
  if (rc) return rc;
  rc = check_rank_comm(c, e);
  if (rc) return rc;
  if (!out_score_dev || !out_row_dev) return fail(SA_ERR_ARG, "null buffer");
  SA_ON_DEVICE(e->device);
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  SA_CUDA(cudaStreamWaitEvent(st, e->scratch_free, 0));
  return sharded_search_on_stream(c, 0, e, q_bf16_dev, nq, k, row_offset, out_score_dev,
                                  reinterpret_cast<long long*>(out_row_dev), st, 7,
                                  reinterpret_cast<const sa::Filter*>(filters_dev));
}

int sa_sharded_search(sa_comm* c, sa_engine* e, const void* q_bf16_dev, int nq, int k, int64_t row_offset,
                      float* out_score_dev, int64_t* out_row_dev, uintptr_t stream) {
  return sharded_search(c, e, q_bf16_dev, nullptr, false, nq, k, row_offset, out_score_dev, out_row_dev, stream);
}

int sa_sharded_search_filtered(sa_comm* c, sa_engine* e, const void* q_bf16_dev, const sa_filter* filters_dev, int nq,
                               int k, int64_t row_offset, float* out_score_dev, int64_t* out_row_dev, uintptr_t stream) {
  return sharded_search(c, e, q_bf16_dev, filters_dev, true, nq, k, row_offset, out_score_dev, out_row_dev, stream);
}

static int sharded_search_host_submit(sa_comm* c, sa_engine* e, int slot, const float* q_f32_host,
                                      const sa_filter* filters_host, bool filtered, int nq, int k, int64_t row_offset) {
  int rc = check_search(e, filters_host, filtered);
  if (rc) return rc;
  rc = check_rank_comm(c, e);
  if (rc) return rc;
  if (slot < 0 || slot >= kHostSlots) return fail(SA_ERR_ARG, "slot %d outside [0, %d)", slot, kHostSlots);
  return host_submit(e, slot, q_f32_host, nq, k, c, 0, row_offset, 7, filters_host);
}

int sa_sharded_search_host_submit(sa_comm* c, sa_engine* e, int slot, const float* q_f32_host, int nq, int k,
                                  int64_t row_offset) {
  return sharded_search_host_submit(c, e, slot, q_f32_host, nullptr, false, nq, k, row_offset);
}

int sa_sharded_search_host_submit_filtered(sa_comm* c, sa_engine* e, int slot, const float* q_f32_host,
                                           const sa_filter* filters_host, int nq, int k, int64_t row_offset) {
  return sharded_search_host_submit(c, e, slot, q_f32_host, filters_host, true, nq, k, row_offset);
}

int sa_sharded_search_host_wait(sa_comm* c, sa_engine* e, int slot, float* out_score_host, int64_t* out_row_host) {
  int rc = check_engine(e);
  if (rc) return rc;
  if (!c) return fail(SA_ERR_ARG, "null communicator");
  if (slot < 0 || slot >= kHostSlots) return fail(SA_ERR_ARG, "slot %d outside [0, %d)", slot, kHostSlots);
  return host_wait(e, slot, out_score_host, out_row_host, true);
}

static int gather_merge_submit(sa_comm* c, sa_engine* const* engines, int slot, const float* q_f32_host,
                               const sa_filter* filters_host, int nq, int k, const int64_t* shard_offsets) {
  if (!c || !engines || !shard_offsets) return fail(SA_ERR_ARG, "null argument");
  if (c->rank >= 0) return fail(SA_ERR_ARG, "multi-process communicator: use sa_sharded_search*");
  if (slot < 0 || slot >= kHostSlots) return fail(SA_ERR_ARG, "slot %d outside [0, %d)", slot, kHostSlots);
  for (int g = 0; g < c->n_ranks; ++g) {
    int rc = check_engine(engines[g]);
    if (rc) return rc;
    if (engines[g]->device != c->devices[g])
      return fail(SA_ERR_ARG, "engine %d is on device %d, communicator rank %d on %d", g, engines[g]->device, g, c->devices[g]);
    if (engines[g]->sim != engines[0]->sim)
      return fail(SA_ERR_ARG, "engine %d has similarity %d, engine 0 has %d", g, engines[g]->sim, engines[0]->sim);
    if (engines[g]->elem != engines[0]->elem)
      return fail(SA_ERR_ARG, "engine %d has element type %d, engine 0 has %d", g, engines[g]->elem, engines[0]->elem);
    if (filters_host != nullptr) {
      rc = check_filtered(engines[g], filters_host);
      if (rc) return rc;
    }
  }
  // every GPU gets the query block and runs the identical single-GPU path; the collectives of all local ranks are
  // issued inside one NCCL group (a single thread drives all devices)
  int rc = SA_OK;
  for (int g = 0; g < c->n_ranks; ++g) {
    rc = host_submit(engines[g], slot, q_f32_host, nq, k, c, g, shard_offsets[g], 1, filters_host);
    if (rc) return rc;
  }
  SA_NCCL(g_nccl.GroupStart());
  for (int g = 0; g < c->n_ranks && rc == SA_OK; ++g)
    rc = host_submit(engines[g], slot, q_f32_host, nq, k, c, g, shard_offsets[g], 2);
  ncclResult_t r = g_nccl.GroupEnd();
  if (rc) return rc;
  if (r != ncclSuccess) return fail(SA_ERR_COMM, "ncclGroupEnd failed: %s", g_nccl.GetErrorString(r));
  for (int g = 0; g < c->n_ranks; ++g) {
    rc = host_submit(engines[g], slot, q_f32_host, nq, k, c, g, shard_offsets[g], 4);
    if (rc) return rc;
  }
  return SA_OK;
}

int sa_gather_merge_submit(sa_comm* c, sa_engine* const* engines, int slot, const float* q_f32_host, int nq, int k,
                           const int64_t* shard_offsets) {
  return gather_merge_submit(c, engines, slot, q_f32_host, nullptr, nq, k, shard_offsets);
}

int sa_gather_merge_submit_filtered(sa_comm* c, sa_engine* const* engines, int slot, const float* q_f32_host,
                                    const sa_filter* filters_host, int nq, int k, const int64_t* shard_offsets) {
  if (!filters_host) return fail(SA_ERR_ARG, "null filters");
  return gather_merge_submit(c, engines, slot, q_f32_host, filters_host, nq, k, shard_offsets);
}

int sa_gather_merge_wait(sa_comm* c, sa_engine* const* engines, int slot, float* out_score_host, int64_t* out_row_host) {
  if (!c || !engines) return fail(SA_ERR_ARG, "null argument");
  if (slot < 0 || slot >= kHostSlots) return fail(SA_ERR_ARG, "slot %d outside [0, %d)", slot, kHostSlots);
  // every rank holds the same merged answer; hand out rank 0's and retire the other slots
  int rc = host_wait(engines[0], slot, out_score_host, out_row_host, true);
  for (int g = 1; g < c->n_ranks; ++g) {
    sa_engine::HostSlot& sl = engines[g]->slot[slot];
    if (sl.busy) {
      DeviceGuard dg(engines[g]->device);
      cudaEventSynchronize(sl.done);
      sl.busy = false;
    }
  }
  return rc;
}

int sa_gather_merge(sa_comm* c, sa_engine* const* engines, const float* q_f32_host, int nq, int k,
                    const int64_t* shard_offsets, float* out_score_host, int64_t* out_row_host) {
  int rc = sa_gather_merge_submit(c, engines, 0, q_f32_host, nq, k, shard_offsets);
  if (rc) return rc;
  return sa_gather_merge_wait(c, engines, 0, out_score_host, out_row_host);
}

int sa_gather_merge_filtered(sa_comm* c, sa_engine* const* engines, const float* q_f32_host, const sa_filter* filters_host,
                             int nq, int k, const int64_t* shard_offsets, float* out_score_host, int64_t* out_row_host) {
  int rc = sa_gather_merge_submit_filtered(c, engines, 0, q_f32_host, filters_host, nq, k, shard_offsets);
  if (rc) return rc;
  return sa_gather_merge_wait(c, engines, 0, out_score_host, out_row_host);
}

namespace {
// Event times of the search `back` positions before the newest one (0 = newest).  Synchronises on its last event.
int read_timing(sa_engine* e, int back, float* scan_ms, float* total_ms, const sa_engine::Timing** out) {
  if (e->n_searches <= back || back >= kTimingRing) return fail(SA_ERR_ARG, "no such search in the timing ring");
  const sa_engine::Timing& tm = e->ring[(e->n_searches - 1 - back) % kTimingRing];
  SA_CUDA(cudaEventSynchronize(tm.ev_total[1]));
  float tot = 0.f, scan = 0.f;
  SA_CUDA(cudaEventElapsedTime(&tot, tm.ev_total[0], tm.ev_total[1]));
  for (int i = 0; i < tm.launches; ++i) {
    float ms = 0.f;
    SA_CUDA(cudaEventElapsedTime(&ms, tm.ev_scan[i][0], tm.ev_scan[i][1]));
    scan += ms;
  }
  *scan_ms = scan;
  *total_ms = tot;
  *out = &tm;
  return SA_OK;
}
}  // namespace

int sa_last_timing(sa_engine* e, float* scan_ms, float* total_ms, double* bytes, double* flops, int* launches,
                   int* kernels) {
  if (!e) return fail(SA_ERR_ARG, "null engine");
  if (e->n_searches == 0) return fail(SA_ERR_ARG, "no search has run on this engine");
  SA_ON_DEVICE(e->device);
  float scan = 0.f, tot = 0.f;
  const sa_engine::Timing* tm = nullptr;
  int rc = read_timing(e, 0, &scan, &tot, &tm);
  if (rc) return rc;
  if (scan_ms) *scan_ms = scan;
  if (total_ms) *total_ms = tot;
  if (bytes) *bytes = tm->bytes;
  if (flops) *flops = tm->flops;
  if (launches) *launches = tm->launches;
  if (kernels) *kernels = tm->kernels;
  return SA_OK;
}

int sa_timing_mean(sa_engine* e, int n, float* scan_ms_mean, float* total_ms_mean, int* n_used) {
  if (!e || !scan_ms_mean || !total_ms_mean || !n_used) return fail(SA_ERR_ARG, "null argument");
  if (e->n_searches == 0) return fail(SA_ERR_ARG, "no search has run on this engine");
  SA_ON_DEVICE(e->device);
  const int m = static_cast<int>(std::min<long long>(std::min(n, kTimingRing), e->n_searches));
  if (m <= 0) return fail(SA_ERR_ARG, "n must be positive");
  double ssum = 0, tsum = 0;
  for (int b = 0; b < m; ++b) {
    float scan = 0.f, tot = 0.f;
    const sa_engine::Timing* tm = nullptr;
    int rc = read_timing(e, b, &scan, &tot, &tm);
    if (rc) return rc;
    ssum += scan;
    tsum += tot;
  }
  *scan_ms_mean = static_cast<float>(ssum / m);
  *total_ms_mean = static_cast<float>(tsum / m);
  *n_used = m;
  return SA_OK;
}

namespace {
// Options of sa_set_option: the engine field each sets and the values it accepts.  A flag accepts any value and stores
// 1 for a nonzero one; any other option accepts [lo, hi].
using EngineField = int sa_engine::*;
struct EngineOption {
  const char* name;
  EngineField field;
  bool flag;
  int64_t lo = 0, hi = 0;
};
constexpr EngineOption kOptions[] = {
    {"cta_group", &sa_engine::opt_cta_group, false, 0, 2},
    {"unit_map", &sa_engine::opt_unit_map, false, 0, 1},
    {"wait_hint_ns", &sa_engine::opt_wait_hint_ns, false, -1, 1000000},
    {"presample", &sa_engine::opt_presample, false, -1, 4096},
    {"pace_gain", &sa_engine::opt_pace_gain, false, -1, 4096},
    {"pace_max", &sa_engine::opt_pace_max, false, -1, 65536},
    {"max_drift", &sa_engine::opt_max_drift, false, -1, 1024},
    {"max_launch_qblocks", &sa_engine::opt_max_launch_qblocks, false, 0, INT_MAX},
    {"force_fix", &sa_engine::opt_force_fix, true},
    {"count_fix", &sa_engine::opt_count_fix, true},
    {"profile", &sa_engine::opt_profile, true},
    {"share_thresholds", &sa_engine::opt_share_thresholds, true},
    {"window_bound", &sa_engine::opt_window_bound, true},
    {"record_times", &sa_engine::opt_record_times, true},
};
}  // namespace

int sa_set_option(sa_engine* e, const char* name, int64_t value) {
  if (!e || !name) return fail(SA_ERR_ARG, "null argument");
  if (!strcmp(name, "list_len")) {  // the one option whose values are a set rather than a range
    if (value != 0 && value != 16 && value != 32) return fail(SA_ERR_ARG, "list_len must be 0, 16 or 32");
    e->opt_list_len = static_cast<int>(value);
    return SA_OK;
  }
  for (const EngineOption& o : kOptions) {
    if (strcmp(name, o.name)) continue;
    if (o.flag) {
      e->*o.field = value != 0;
      return SA_OK;
    }
    if (value < o.lo || value > o.hi)
      return fail(SA_ERR_ARG, "%s must be in [%lld, %lld]", name, static_cast<long long>(o.lo),
                  static_cast<long long>(o.hi));
    e->*o.field = static_cast<int>(value);
    return SA_OK;
  }
  return fail(SA_ERR_ARG, "unknown option '%s'", name);
}

int sa_get_info(const sa_engine* e, const char* name, int64_t* value) {
  if (!e || !name || !value) return fail(SA_ERR_ARG, "null argument");
  if (!strcmp(name, "num_sms")) *value = e->num_sms;
  else if (!strcmp(name, "dim")) *value = e->dim;
  else if (!strcmp(name, "capacity")) *value = e->capacity;
  else if (!strcmp(name, "n_rows")) *value = e->n_rows;
  else if (!strcmp(name, "max_batch")) *value = e->max_batch;
  else if (!strcmp(name, "max_k")) *value = e->max_k;
  else if (!strcmp(name, "last_grid")) *value = e->last_grid;
  else if (!strcmp(name, "dbg_times_ptr")) *value = static_cast<int64_t>(reinterpret_cast<uintptr_t>(e->dbg_times));
  else if (!strcmp(name, "last_fix_entries")) *value = e->last_fix_entries;
  else if (!strcmp(name, "eps_rel_e12"))
    *value = static_cast<int64_t>(static_cast<double>(scan_eps_rel(e->dim, e->elem)) * 1e12);
  else if (!strcmp(name, "similarity")) *value = e->sim;
  else if (!strcmp(name, "elem")) *value = e->elem;
  else if (!strcmp(name, "has_tags")) *value = e->row_tags != nullptr ? 1 : 0;
  else if (!strcmp(name, "cmax_bits")) {
    unsigned bits = 0;
    DeviceGuard dg(e->device);
    if (cudaMemcpy(&bits, e->cmax, sizeof bits, cudaMemcpyDeviceToHost) != cudaSuccess)
      return fail(SA_ERR_CUDA, "reading cmax failed");
    *value = bits;
  }
  else return fail(SA_ERR_ARG, "unknown info '%s'", name);
  return SA_OK;
}

int sa_scan_profile(sa_engine* e, int64_t* out_host, int max_ctas, int* n_ctas) {
  if (!e || !out_host || !n_ctas) return fail(SA_ERR_ARG, "null argument");
  static_assert(sizeof(sa::ScanProf) == 8 * sizeof(int64_t), "profile record is 8 x int64");
  SA_ON_DEVICE(e->device);
  const int n = std::min(std::min(max_ctas, e->last_grid), e->num_sms);
  SA_CUDA(cudaDeviceSynchronize());
  SA_CUDA(cudaMemcpy(out_host, e->prof, static_cast<size_t>(n) * sizeof(sa::ScanProf), cudaMemcpyDeviceToHost));
  *n_ctas = n;
  return SA_OK;
}

int sa_debug_tile_dots(sa_engine* e, const void* q_bf16_dev, int nq, int tile, int cta_group, float* out_dots_dev,
                       uintptr_t stream) {
  int rc = check_engine(e);
  if (rc) return rc;
  if (!q_bf16_dev || !out_dots_dev) return fail(SA_ERR_ARG, "null buffer");
  if (cta_group != 1 && cta_group != 2) return fail(SA_ERR_ARG, "cta_group must be 1 or 2");
  const int num_tiles = static_cast<int>((e->n_rows + sa::kBlockN - 1) / sa::kBlockN);
  if (tile < 0 || tile >= num_tiles) return fail(SA_ERR_ARG, "tile %d outside [0, %d)", tile, num_tiles);
  const int rows_per_qb = 128 * cta_group;
  const int nqb = (nq + rows_per_qb - 1) / rows_per_qb;
  if (nq <= 0 || nqb * cta_group > e->num_sms) return fail(SA_ERR_CAPACITY, "nq too large for the debug hook");
  SA_ON_DEVICE(e->device);
  CUtensorMap tq;
  rc = encode_rows_map(&tq, q_bf16_dev, static_cast<uint64_t>(nq), e->dim, sa::kBlockM, e->elem);
  if (rc) return rc;
  sa::ScanParams sp = {};
  sp.row_term = e->row_term;
  sp.n_rows = e->n_rows;
  sp.nq = nq;
  sp.num_kb = e->dim * sa::elem_bytes(e->elem) / 128;  // 128-byte K slices
  sp.num_tiles = num_tiles;
  sp.nqb = nqb;
  sp.tl_count = 1;  // one tile lane: every unit walks all tiles, dumps `tile`
  sp.part_score = e->part_score;
  sp.part_idx = e->part_idx;
  sp.part_drop = e->part_drop;
  sp.tile_stride = 1;
  sp.dbg_dots = out_dots_dev;
  sp.dbg_tile = tile;
  const int epi = sa::kEpiMul | (e->elem == SA_ELEM_INT8 ? sa::kEpiI8 : 0);
  return launch_scan_dispatch(cta_group, 16, sa::kModeDots, epi, tq, e->tmap_c[cta_group - 1], sp, nqb * cta_group,
                              reinterpret_cast<cudaStream_t>(stream));
}

int sa_debug_plan(int num_sms, int nq, int cta_group, int num_tiles, int max_launch_qblocks, int* out, int max_out,
                  int* n_launches) {
  if (!out || !n_launches) return fail(SA_ERR_ARG, "null argument");
  if (num_sms < 2 || nq <= 0 || num_tiles < 0 || (cta_group != 1 && cta_group != 2))
    return fail(SA_ERR_ARG, "bad planning input");
  std::vector<LaunchPlan> plan = plan_search(num_sms, max_launch_qblocks, nq, cta_group, std::max(num_tiles, 1));
  if (static_cast<int>(plan.size()) > max_out) return fail(SA_ERR_CAPACITY, "plan has %zu launches", plan.size());
  for (size_t i = 0; i < plan.size(); ++i) {
    out[4 * i + 0] = plan[i].q0;
    out[4 * i + 1] = plan[i].nq;
    out[4 * i + 2] = plan[i].nqb;
    out[4 * i + 3] = plan[i].tl;
  }
  *n_launches = static_cast<int>(plan.size());
  return SA_OK;
}

// ---- host-side test hooks over the pure device helpers (compiled __host__ __device__; no GPU involved) ----------
int sa_debug_float_keys(const float* x, int n, uint32_t* key, float* back, float* below) {
  if (!x || !key || !back || !below || n < 0) return fail(SA_ERR_ARG, "bad argument");
  for (int i = 0; i < n; ++i) {
    key[i] = sa::float_to_key(x[i]);
    back[i] = sa::key_to_float(key[i]);
    below[i] = sa::float_below(x[i]);
  }
  return SA_OK;
}

int sa_debug_bf16_round(const float* x, int n, uint16_t* bits, float* back) {
  if (!x || !bits || !back || n < 0) return fail(SA_ERR_ARG, "bad argument");
  for (int i = 0; i < n; ++i) {
    bits[i] = static_cast<uint16_t>(sa::f32_to_bf16_bits(x[i]));
    back[i] = sa::bf16_bits_to_f32(bits[i]);
  }
  return SA_OK;
}

int sa_debug_int8_round(const float* x, int n, int8_t* out) {
  if (!x || !out || n < 0) return fail(SA_ERR_ARG, "bad argument");
  for (int i = 0; i < n; ++i) out[i] = static_cast<int8_t>(sa::f32_to_i8(x[i]));
  return SA_OK;
}

int sa_debug_merge_keys(const float* score, const int32_t* row, int n, uint64_t* key, int32_t* row_back) {
  if (!score || !row || !key || !row_back || n < 0) return fail(SA_ERR_ARG, "bad argument");
  for (int i = 0; i < n; ++i) {
    key[i] = sa::make_key(score[i], row[i]);
    row_back[i] = sa::key_row(key[i]);
  }
  return SA_OK;
}

int sa_debug_list_insert(const float* score, const int32_t* row, int n, int list_len, const float* floor_after,
                         float* out_score, int32_t* out_row, float* out_drop) {
  if (!score || !row || !out_score || !out_row || n < 0) return fail(SA_ERR_ARG, "bad argument");
  if (list_len == 16) run_list<16>(score, row, n, floor_after, out_score, out_row, out_drop);
  else if (list_len == 32) run_list<32>(score, row, n, floor_after, out_score, out_row, out_drop);
  else return fail(SA_ERR_ARG, "list_len must be 16 or 32");
  return SA_OK;
}

int sa_debug_window_bound(const uint32_t* keys, int n_windows, int list_len, uint32_t* out_bound, uint32_t* out_sorted) {
  if (!keys || !out_bound || n_windows < 0) return fail(SA_ERR_ARG, "bad argument");
  if (list_len != 16 && list_len != 32) return fail(SA_ERR_ARG, "list_len must be 16 or 32");
  for (int w = 0; w < n_windows; ++w) {
    unsigned x[sa::kWin];
    for (int i = 0; i < sa::kWin; ++i) x[i] = keys[static_cast<size_t>(w) * sa::kWin + i];
    out_bound[w] = list_len == 16 ? sa::window_bound<16>(x) : sa::window_bound<32>(x);
    if (out_sorted)
      for (int i = 0; i < sa::kWin; ++i) out_sorted[static_cast<size_t>(w) * sa::kWin + i] = x[i];
  }
  return SA_OK;
}

int sa_debug_window_bound_deep(const uint32_t* keys, int n_windows, uint32_t* out_bound) {
  if (!keys || !out_bound || n_windows < 0) return fail(SA_ERR_ARG, "bad argument");
  for (int w = 0; w < n_windows; ++w) {
    unsigned x[sa::kWin];
    for (int i = 0; i < sa::kWin; ++i) x[i] = keys[static_cast<size_t>(w) * sa::kWin + i];
    out_bound[w] = sa::window_bound<32, true>(x);
  }
  return SA_OK;
}

int sa_debug_filter_pass(const uint64_t* tags, int n, const sa_filter* f, uint8_t* out) {
  if (!tags || !f || !out || n < 0) return fail(SA_ERR_ARG, "bad argument");
  const sa::Filter& F = *reinterpret_cast<const sa::Filter*>(f);
  for (int i = 0; i < n; ++i) out[i] = sa::filter_pass(tags[i], F) ? 1 : 0;
  return SA_OK;
}

int sa_host_alloc(void** out, uint64_t bytes) {
  if (!out) return fail(SA_ERR_ARG, "null out");
  SA_CUDA(cudaHostAlloc(out, bytes, cudaHostAllocDefault));
  return SA_OK;
}

int sa_host_free(void* p) {
  SA_CUDA(cudaFreeHost(p));
  return SA_OK;
}

}  // extern "C"
