// api.cu — C ABI of libluxb (include/lux_b200.h) and the thin per-rank host runtime behind it.
// Replaces, for the hot path only: Graph::Graph + load/scan/init tasks, pull_app_task_impl / push_app_task_impl,
// the app driver loops and LuxMapper's placement (see the citations in lux_b200.h).
// Product code: nothing here may include, link or call oracle/.
#include <cub/cub.cuh>
#include <stdarg.h>
#include <stdlib.h>
#include <string.h>
#include <algorithm>
#include <type_traits>
#include <new>

#include "build.cuh"
#include "cf.cuh"
#include "pull.cuh"
#include "panel.cuh"
#include "seg.cuh"
#include "push.cuh"
#include "runtime.cuh"
#include <thrust/iterator/counting_iterator.h>

using namespace luxb;

// How an app runs: luxb_iterate for a fixed number of iterations, luxb_run_to_convergence, or an entry point of its own
enum class AppRun : uint8_t { kIterations, kConvergence, kEntry };
static constexpr char kBcRun[] = "luxb_bc_run";  // betweenness centrality, over hop levels or weighted distance classes

// One row per luxb_app: what the runtime asks about an app outside the switches that run its work
struct AppInfo {
  const char* name;  // in messages
  AppRun run;
  const char* entry;  // AppRun::kEntry: the entry point that runs it
  bool weights;       // reads the CSC's edge weights
  // labels are weighted distances (u32, INF = LUXB_DIST_INF, label_iteration<WeightedDistProgram>): the app keeps out_w
  // beside the push CSR and pulls through the merge-path sweep only
  bool dist_labels;
  uint32_t vbytes;  // bytes per vertex value
  bool check;       // luxb_check applies
  bool settable;    // luxb_set_values / luxb_set_local_values apply
};
static constexpr AppInfo kApps[] = {
    // name                             run                   entry             weights dist   vbytes    check  settable
    {"pagerank",                        AppRun::kIterations,  nullptr,          false,  false, 4,        false, true},
    {"connected components",            AppRun::kConvergence, nullptr,          false,  false, 4,        true,  true},
    {"SSSP",                            AppRun::kConvergence, nullptr,          false,  false, 4,        true,  true},
    {"col_filter",                      AppRun::kIterations,  nullptr,          true,   false, 4 * kCfK, false, true},
    {"weighted SSSP",                   AppRun::kConvergence, nullptr,          true,   true,  4,        true,  true},
    {"betweenness centrality",          AppRun::kEntry,       kBcRun,           false,  false, 8,        false, true},
    {"weighted betweenness centrality", AppRun::kEntry,       kBcRun,           true,   true,  8,        false, true},
    {"triangle counting",               AppRun::kEntry,       "luxb_tc_run",    false,  false, 8,        false, false},
    {"k-core decomposition",            AppRun::kEntry,       "luxb_kcore_run", false,  false, 4,        true,  true},
    {"k-truss decomposition",           AppRun::kEntry,       "luxb_truss_run", false,  false, 4,        true,  false},
};
static constexpr int kNumApps = sizeof(kApps) / sizeof(kApps[0]);
static_assert(kNumApps == LUXB_TRUSS + 1, "one row per luxb_app");
// the handle's app (its config passed check_config at open)
static const AppInfo& app_of(const luxb_graph* g) { return kApps[g->cfg.app]; }

// 0 .. 11: phases of the compute stream (the concurrent sweep's side stream adds to pull_tile, fixup and cold_hub);
// 12 .. 14: the concurrent sweep's main kernel on the panel's SMs, the wait for the side stream, the whole overlapped region
static const char* const kPhaseName[15] = {"pull_tile", "fixup", "refresh", "rechunk", "barrier", "panel", "combine", "pack+push",
                                           "pull/bcast", "cold_hub", "bc_sigma", "bc_delta", "main_join", "join_wait", "overlap"};
static void pt_mark(luxb_graph* g, int tag) {
  PhaseTimer& pt = g->pt;
  if (!pt.on) return;
  cudaEvent_t e;
  cudaEventCreate(&e);
  cudaEventRecord(e, g->stream);
  pt.ev.push_back(e);
  pt.tag.push_back(tag);
}
// an event on stream st for pt_span: its index, or -1 when the timer is off
static int pt_event(luxb_graph* g, cudaStream_t st) {
  PhaseTimer& pt = g->pt;
  if (!pt.on) return -1;
  cudaEvent_t e;
  cudaEventCreate(&e);
  cudaEventRecord(e, st);
  pt.span_ev.push_back(e);
  return (int)pt.span_ev.size() - 1;
}
static void pt_span(luxb_graph* g, int tag, int begin, int end) {
  if (begin >= 0) g->pt.spans.push_back({begin, end, tag});
}
static void pt_print(luxb_graph* g) {
  if (g->pt.on && g->pt.cnt) {
    char line[1024];
    // betweenness centrality times its two level sweeps per source (the BFS before them is not split)
    const bool bc = app_of(g).entry == kBcRun;
    int n = snprintf(line, sizeof(line), "[luxb rank %d] phase means over %ld %s:", g->cfg.rank, g->pt.cnt, bc ? "sources" : "iterations");
    double sum = 0;
    for (int k = bc ? 10 : 0; k < (bc ? 12 : 10); ++k) {
      n += snprintf(line + n, sizeof(line) - n, " %s %.3f ms;", kPhaseName[k], g->pt.sum[k] / g->pt.cnt);
      sum += g->pt.sum[k] / g->pt.cnt;
    }
    if (!bc && g->pt.sum[14] > 0) {  // concurrent sweep: the phases above overlap, the compute stream's total is the time
      for (int k = 12; k < 15; ++k) n += snprintf(line + n, sizeof(line) - n, " %s %.3f ms;", kPhaseName[k], g->pt.sum[k] / g->pt.cnt);
      sum = g->pt.chain / g->pt.cnt;
    }
    snprintf(line + n, sizeof(line) - n, " sum %.3f ms\n", sum);
    fputs(line, stderr);  // one write per rank: the ranks' lines do not interleave
  }
}

static void pt_flush(luxb_graph* g) {
  PhaseTimer& pt = g->pt;
  if (!pt.on || pt.ev.empty()) return;
  cudaStreamSynchronize(g->stream);  // the side stream joins the compute stream before every sweep ends
  // one PageRank iteration (its pull sweep), or one BC source (its σ sweep: the BFS's own pull sweeps also mark tag 0)
  const int count_tag = app_of(g).entry == kBcRun ? 10 : 0;
  for (size_t i = 1; i < pt.ev.size(); ++i) {
    if (pt.tag[i] < 0) continue;
    float ms = 0;
    cudaEventElapsedTime(&ms, pt.ev[i - 1], pt.ev[i]);
    pt.sum[pt.tag[i]] += ms;
    pt.chain += ms;
    if (pt.tag[i] == count_tag) pt.cnt++;
  }
  for (const PhaseTimer::Span& s : pt.spans) {
    float ms = 0;
    cudaEventElapsedTime(&ms, pt.span_ev[s.begin], pt.span_ev[s.end]);
    pt.sum[s.tag] += ms;
    if (s.tag == count_tag) pt.cnt++;
  }
  for (cudaEvent_t e : pt.ev) cudaEventDestroy(e);
  for (cudaEvent_t e : pt.span_ev) cudaEventDestroy(e);
  pt.ev.clear();
  pt.tag.clear();
  pt.span_ev.clear();
  pt.spans.clear();
}


// ------------------------------------------------------------------------------------------------------------
namespace luxb {
static thread_local char g_err[1024] = "";
void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}
}  // namespace luxb

#define LUXB_ARG(cond, ...)             \
  do {                                  \
    if (!(cond)) {                      \
      set_error(__VA_ARGS__);           \
      return LUXB_ERR_ARG;              \
    }                                   \
  } while (0)

#define LUXB_NCCL(expr)                                                                              \
  do {                                                                                               \
    ncclResult_t _r = (expr);                                                                        \
    if (_r != ncclSuccess) {                                                                         \
      set_error("NCCL error %s at %s:%d: %s", #expr, __FILE__, __LINE__, nccl().GetErrorString(_r)); \
      return LUXB_ERR_COMM;                                                                          \
    }                                                                                                \
  } while (0)

// merge-path shapes <items per lane, consumer warps per CTA, ring stages>; chosen at open time (LUXB_PULL_SHAPE).
// Shared memory is kept small on purpose: what the ring does not take stays L1, and the gather rate follows L1 size.
#define LUXB_PULL_SHAPES(X) X(0, 7, 8, 2) X(1, 9, 8, 2) X(2, 7, 16, 2)
#define LUXB_DECL_SHAPE(id, ipt, warps, stages) using PullShape##id = PullShape<ipt, warps, stages>;
LUXB_PULL_SHAPES(LUXB_DECL_SHAPE)
#define LUXB_TILE_OF(id, ipt, warps, stages) PullShape##id::kTile,
static const int kPullTileOf[] = {LUXB_PULL_SHAPES(LUXB_TILE_OF)};
static const int kNumPullShapes = sizeof(kPullTileOf) / sizeof(int);
static const int kDefaultPullShape = 0;
static const int kDefaultPullCtas = 3;

static inline int grid_for(uint64_t n, int threads, int cap) {
  uint64_t b = (n + threads - 1) / threads;
  if (b < 1) b = 1;
  if (b > (uint64_t)cap) b = cap;
  return (int)b;
}

// every buffer is padded: at least one element, plus 256 bytes
template <class T>
static size_t padded_bytes(uint64_t count) { return std::max<uint64_t>(count, 1) * sizeof(T) + 256; }

// The one allocator of the buffers the graph keeps: each is recorded in g->owned, which luxb_close frees in reverse
template <class T>
static int gmalloc(luxb_graph* g, T** p, uint64_t count, MemKind kind = MemKind::kDevice) {
  void* q = nullptr;
  if (kind == MemKind::kDevice) LUXB_CUDA(cudaMalloc(&q, padded_bytes<T>(count)));
  else if (kind == MemKind::kPinned) LUXB_CUDA(cudaMallocHost(&q, padded_bytes<T>(count)));
  else LUXB_CUDA(cudaHostAlloc(&q, padded_bytes<T>(count), cudaHostAllocMapped | cudaHostAllocPortable));
  g->owned.push_back({q, kind});
  *p = reinterpret_cast<T*>(q);
  return 0;
}

static cudaError_t free_owned(const OwnedBuf& b) { return b.kind == MemKind::kDevice ? cudaFree(b.p) : cudaFreeHost(b.p); }

// free one of the graph's buffers before luxb_close
static int gfree(luxb_graph* g, void* p) {
  for (size_t i = 0; i < g->owned.size(); ++i)
    if (g->owned[i].p == p) {
      const OwnedBuf b = g->owned[i];
      g->owned.erase(g->owned.begin() + i);
      LUXB_CUDA(free_owned(b));
      return 0;
    }
  return 0;
}

// edge arrays: HBM, or mapped pinned host memory when cfg.zero_copy_edges (TMA bulk copies and plain loads read it
// over PCIe through the same unified addresses)
template <class T>
static int edge_alloc(luxb_graph* g, T** p, uint64_t count) {
  return gmalloc(g, p, count, g->cfg.zero_copy_edges ? MemKind::kMapped : MemKind::kDevice);
}

// temporaries of a build step: freed on every exit path
struct DevTmp {
  std::vector<void*> ptrs;
  ~DevTmp() { for (void* q : ptrs) cudaFree(q); }
  template <class T>
  int alloc(T** out, uint64_t count) {
    void* q = nullptr;
    LUXB_CUDA(cudaMalloc(&q, padded_bytes<T>(count)));
    ptrs.push_back(q);
    *out = reinterpret_cast<T*>(q);
    return 0;
  }
  void release(void* q) {
    for (size_t i = 0; i < ptrs.size(); ++i)
      if (ptrs[i] == q) { cudaFree(q); ptrs.erase(ptrs.begin() + i); return; }
  }
  void keep(luxb_graph* g, void* q) {  // ownership moves to the graph
    for (size_t i = 0; i < ptrs.size(); ++i)
      if (ptrs[i] == q) { ptrs.erase(ptrs.begin() + i); g->owned.push_back({q, MemKind::kDevice}); return; }
  }
};

// one two-phase cub call f(temp, bytes) on `stream`: size query, temporary storage from `tmp`, the call; the storage is
// released once the stream has finished with it
template <class F>
static int cub_call(DevTmp& tmp, cudaStream_t stream, F&& f) {
  size_t bytes = 0;
  LUXB_CUDA(f(nullptr, bytes));
  char* d_tmp = nullptr;
  LUXB_TRY(tmp.alloc(&d_tmp, bytes));
  LUXB_CUDA(f(d_tmp, bytes));
  LUXB_CUDA(cudaStreamSynchronize(stream));
  tmp.release(d_tmp);
  return 0;
}

// fix-up scratch of a sweep over n_tiles tiles; the fused fix-up adds its chain on first use (launch_fixup)
static int alloc_fixup(luxb_graph* g, FixupScratch& f, uint32_t n_tiles) {
  LUXB_TRY(gmalloc(g, (uint32_t**)&f.d_head, (uint64_t)n_tiles + 1));
  LUXB_TRY(gmalloc(g, (uint32_t**)&f.d_tail, (uint64_t)n_tiles + 1));
  f.n_fix_blocks = (n_tiles + kFixBlock - 1) / kFixBlock;
  LUXB_TRY(gmalloc(g, (uint64_t**)&f.d_carry, (uint64_t)n_tiles + 1));
  LUXB_TRY(gmalloc(g, &f.d_carry_flag, (uint64_t)n_tiles + 1));
  LUXB_TRY(gmalloc(g, (uint64_t**)&f.d_block_agg, (uint64_t)f.n_fix_blocks + 1));
  LUXB_TRY(gmalloc(g, &f.d_block_flag, (uint64_t)f.n_fix_blocks + 1));
  return 0;
}

// ---- the reference partitioner on the host (pull_model.inl:108-131); same cut rule as partition_kernel -------
static int host_partition(uint32_t nv, uint64_t ne, const uint64_t* row_end, int P, uint32_t* rl, uint32_t* np,
                          uint64_t* cl) {
  uint64_t cap = (ne + P - 1) / P;
  uint32_t left = 0;
  int count = 0, found_adjust = 0;
  while (left < nv && count < P) {
    uint64_t base = left == 0 ? 0 : row_end[left - 1];
    const uint64_t* first = std::upper_bound(row_end + left, row_end + nv, base + cap);  // first row_end[v] > base+cap
    uint32_t v = (uint32_t)(first - row_end);
    if (v < nv) {
      rl[count] = left; np[count] = v - left + 1; cl[count] = base; ++count;
      left = v + 1;
    } else {
      // the reference emits the remainder only if it holds edges (pull_model.inl:128-130) and would then assert
      // on the partition count; we always keep trailing zero-in-degree vertices so that none is dropped
      if (row_end[nv - 1] - base == 0) --found_adjust;
      rl[count] = left; np[count] = nv - left; cl[count] = base; ++count;
      left = nv;
    }
  }
  int found = count + found_adjust;
  for (int p = count; p < P; ++p) { rl[p] = nv; np[p] = 0; cl[p] = ne; }
  return found;
}

// ---- cost-balanced work split (cfg.balanced_split, pull apps) ------------------------------------------------------
// The reference's split balances EDGES; the sweep's cost per edge is not uniform (an edge into a hub destination mostly
// travels through the shared-memory panel, any other edge goes through L1, and every vertex costs bookkeeping; at 8 GPUs
// the reference split gives the last rank 40 % of the RMAT-27 vertices).  Contiguous destination ranges are kept; only
// the cut points move.  Weights in integer units: vertex 8, edge into a hub (in-degree >= kBalanceHubIndeg) 4, other
// edge 7 — fitted on per-rank sweep times of multi-GPU runs of an earlier GPU generation, not re-fitted on H100.
static constexpr uint32_t kBalanceHubIndeg = 64;
static inline uint64_t vertex_cost(uint64_t indeg) { return 8 + (indeg >= kBalanceHubIndeg ? 4 : 7) * indeg; }

static void host_balanced_partition(uint32_t nv, uint64_t ne, const uint64_t* row_end, int P, uint32_t* rl, uint32_t* np, uint64_t* cl) {
  uint64_t total = 0;
  for (uint32_t v = 0; v < nv; ++v) total += vertex_cost(row_end[v] - (v ? row_end[v - 1] : 0));
  uint64_t run = 0;
  uint32_t left = 0;
  int p = 0;
  for (uint32_t v = 0; v < nv && p < P - 1; ++v) {
    run += vertex_cost(row_end[v] - (v ? row_end[v - 1] : 0));
    if (run * P >= total * (uint64_t)(p + 1)) {  // close partition p at v (inclusive)
      rl[p] = left; np[p] = v - left + 1; cl[p] = left ? row_end[left - 1] : 0;
      left = v + 1;
      ++p;
    }
  }
  rl[p] = left; np[p] = nv - left; cl[p] = left ? row_end[left - 1] : 0;
  for (++p; p < P; ++p) { rl[p] = nv; np[p] = 0; cl[p] = ne; }
}

static bool use_balanced_split(const luxb_config* cfg) {
  return cfg->balanced_split && cfg->nranks > 1 && (cfg->app == LUXB_PAGERANK || cfg->app == LUXB_COLFILTER);
}

static int check_config(const luxb_config* cfg) {
  LUXB_ARG(cfg != nullptr, "config is NULL");
  LUXB_ARG((unsigned)cfg->app < (unsigned)kNumApps, "unknown app %d", (int)cfg->app);
  LUXB_ARG(cfg->nranks >= 1 && cfg->nranks <= LUXB_MAX_PARTS, "nranks %d out of range [1,%d]", cfg->nranks, LUXB_MAX_PARTS);
  LUXB_ARG(cfg->rank >= 0 && cfg->rank < cfg->nranks, "rank %d out of range", cfg->rank);
  return 0;
}

static int graph_begin(const luxb_config* cfg, uint32_t nv, uint64_t ne, luxb_graph** out) {
  LUXB_TRY(check_config(cfg));
  LUXB_ARG(out != nullptr, "out is NULL");
  int ndev = 0;
  cudaError_t e = cudaGetDeviceCount(&ndev);
  if (e != cudaSuccess || ndev == 0) {
    set_error("no CUDA device available (%s): libluxb has no CPU fallback", cudaGetErrorString(e));
    return LUXB_ERR_CUDA;
  }
  LUXB_ARG(cfg->device >= 0 && cfg->device < ndev, "device %d out of range (have %d)", cfg->device, ndev);
  LUXB_CUDA(cudaSetDevice(cfg->device));
  luxb_graph* g = new (std::nothrow) luxb_graph();
  if (!g) { set_error("out of host memory"); return LUXB_ERR_NOMEM; }
  g->cfg = *cfg;
  g->P = cfg->nranks;
  g->nv = nv;
  g->ne = ne;
  g->weighted = app_of(g).weights;
  *out = g;
  LUXB_CUDA(cudaStreamCreateWithFlags(&g->stream, cudaStreamNonBlocking));
  LUXB_CUDA(cudaEventCreate(&g->ev_begin));
  LUXB_CUDA(cudaEventCreate(&g->ev_end));
  LUXB_CUDA(cudaDeviceGetAttribute(&g->num_sms, cudaDevAttrMultiProcessorCount, cfg->device));
  g->pull_ctas = kDefaultPullCtas;
  if (const char* env = getenv("LUXB_PULL_CTAS")) g->pull_ctas = std::max(1, atoi(env));
  if (const char* env = getenv("LUXB_PHASE_TIMING")) { g->pt.on = atoi(env) != 0; g->pt.per_call = atoi(env) == 2; }
  if (const char* env = getenv("LUXB_L2_HINTS")) g->l2_hints = atoi(env);
  if (const char* env = getenv("LUXB_OVERLAP")) g->overlap_exchange = atoi(env) != 0;
  if (const char* env = getenv("LUXB_BARRIER")) { g->flag_barrier = strcmp(env, "nccl") != 0; g->flag_barrier_all = strcmp(env, "flag") == 0; }
  if (const char* env = getenv("LUXB_PUSH")) g->direct_push = strcmp(env, "direct") == 0;
  if (const char* env = getenv("LUXB_BARRIER_TIMEOUT_S")) g->barrier_timeout_ns = (uint64_t)std::max(1, atoi(env)) * 1000000000ull;
  if (const char* env = getenv("LUXB_FUSED_FIXUP")) g->fused_fixup = atoi(env) != 0;
  if (const char* env = getenv("LUXB_PANEL_RESERVE_SMS")) g->panel_reserve_sms = std::max(0, atoi(env));
  return 0;
}

static void set_partition_derived(luxb_graph* g) {
  int r = g->cfg.rank;
  g->row_left = g->rl[r];
  g->n_part = g->np[r];
  g->col_left = g->cl[r];
  uint64_t next = (r + 1 < g->P) ? g->cl[r + 1] : g->ne;
  if (g->np[r] == 0) next = g->col_left;
  g->e_part = next - g->col_left;
  uint64_t off = 0;
  for (int p = 0; p < g->P; ++p) {
    uint32_t span = g->np[p] ? g->np[p] - 1 : 0;          // R - L
    g->cap[p] = span / 16 + 100;                          // push_model.inl:393
    g->slot_off[p] = off;
    g->slot_bytes[p] = ((8 + (uint64_t)g->cap[p] * 8) + 15) & ~15ull;  // header + ids + labels
    off += g->slot_bytes[p];
  }
  g->fq_total = off;
}

// the work split is the reference's split (no cfg.balanced_split)
static void use_reference_split(luxb_graph* g) {
  for (int p = 0; p < g->P; ++p) { g->rl[p] = g->ref_rl[p]; g->np[p] = g->ref_np[p]; g->cl[p] = g->ref_cl[p]; }
}

// open of a CSC whose row_end is in host memory: the graph, both splits and this rank's share of them.  On failure the
// caller closes *out if it is set.
static int open_host_begin(const luxb_config* cfg, uint32_t nv, uint64_t ne, const uint64_t* row_end, luxb_graph** out) {
  LUXB_TRY(graph_begin(cfg, nv, ne, out));
  luxb_graph* g = *out;
  g->parts_found = host_partition(nv, ne, row_end, g->P, g->ref_rl, g->ref_np, g->ref_cl);
  if (use_balanced_split(cfg)) host_balanced_partition(nv, ne, row_end, g->P, g->rl, g->np, g->cl);
  else use_reference_split(g);
  set_partition_derived(g);
  return 0;
}

// after d_row_end / d_src are in place: merge-path tile table + per-tile partial buffers
static int finish_layout(luxb_graph* g) {
  uint64_t total = (uint64_t)g->n_part + g->e_part;
  g->pull_shape = kDefaultPullShape;
  if (const char* env = getenv("LUXB_PULL_SHAPE")) {
    int v = atoi(env);
    if (v >= 0 && v < kNumPullShapes) g->pull_shape = v;
  }
  const uint32_t tile = (uint32_t)kPullTileOf[g->pull_shape];
  uint64_t nt = (total + tile - 1) / tile;
  LUXB_ARG(nt < 0xFFFFFFFFull, "partition too large for the tile table");
  PullLayout& B = g->base;
  B.d_row_end = g->d_row_end;
  B.n_vtx = g->n_part;
  B.e_cnt = g->e_part;
  B.n_tiles = (uint32_t)nt;
  LUXB_TRY(gmalloc(g, &B.d_tile_v, (uint64_t)B.n_tiles + 2));
  tile_table_kernel<<<grid_for((uint64_t)B.n_tiles + 1, 256, 1 << 20), 256, 0, g->stream>>>(
      g->d_row_end, g->n_part, g->e_part, tile, B.n_tiles, B.d_tile_v);
  LUXB_CUDA(cudaGetLastError());
  LUXB_TRY(gmalloc(g, &B.d_row_end32, (uint64_t)g->n_part + 8));
  narrow_u64_to_u32_kernel<<<grid_for((uint64_t)g->n_part + 8, 256, 4096), 256, 0, g->stream>>>(g->d_row_end, g->n_part + 4,
                                                                                          B.d_row_end32, (uint64_t)g->n_part + 8);
  LUXB_CUDA(cudaGetLastError());
  LUXB_TRY(alloc_fixup(g, B.fix, B.n_tiles));
  LUXB_TRY(gmalloc(g, &g->d_counters, 8));  // [0] edges scanned, [1] check mistakes, [2] pull tile counter, [3] big segments, [4] panel / cold-hub tile counter
  LUXB_CUDA(cudaMemsetAsync(g->d_counters, 0, 8 * sizeof(unsigned long long), g->stream));
  LUXB_CUDA(cudaStreamSynchronize(g->stream));
  return 0;
}

static int validate_row_end(uint32_t nv, uint64_t ne, const uint64_t* row_end) {
  LUXB_ARG(nv >= 1, "graph has no vertices");
  // device-wide scans / sorts index vertices with 32-bit signed counts and INF = nv must stay a valid label
  LUXB_ARG(nv < 0x7FFFFFFEu, "nv = %u: at most 2^31 - 2 vertices are supported", nv);
  for (uint32_t v = 1; v < nv; ++v)
    LUXB_ARG(row_end[v] >= row_end[v - 1], "row_end not non-decreasing at vertex %u (pull_model.inl:100-101)", v);
  LUXB_ARG(row_end[nv - 1] == ne, "row_end[nv-1] (%llu) != ne (%llu) (pull_model.inl:102)",
           (unsigned long long)row_end[nv - 1], (unsigned long long)ne);
  return 0;
}

// upload this rank's slice given host pointers to ITS portion of row_end (absolute) / src / weight
static int upload_slice(luxb_graph* g, const uint64_t* row_end_slice_abs, const uint32_t* src_slice,
                        const int32_t* weight_slice) {
  LUXB_TRY(gmalloc(g, &g->d_row_end, (uint64_t)g->n_part + 4));
  LUXB_TRY(edge_alloc(g, &g->d_src, g->e_part + 8));
  DevTmp tmp;
  uint64_t* d_tmp = nullptr;
  LUXB_TRY(tmp.alloc(&d_tmp, (uint64_t)g->n_part + 1));
  if (g->n_part)
    LUXB_CUDA(cudaMemcpyAsync(d_tmp, row_end_slice_abs, (size_t)g->n_part * 8, cudaMemcpyHostToDevice, g->stream));
  rowend_rel_kernel<<<grid_for((uint64_t)g->n_part + 4, 256, 4096), 256, 0, g->stream>>>(d_tmp, 0, g->n_part, g->col_left,
                                                                                        g->d_row_end);
  LUXB_CUDA(cudaGetLastError());
  LUXB_CUDA(cudaMemsetAsync(g->d_src, 0, (g->e_part + 8) * 4, g->stream));
  if (g->e_part) LUXB_CUDA(cudaMemcpyAsync(g->d_src, src_slice, g->e_part * 4, cudaMemcpyDefault, g->stream));
  if (g->weighted) {
    LUXB_TRY(edge_alloc(g, &g->d_weight, g->e_part + 8));
    LUXB_CUDA(cudaMemsetAsync(g->d_weight, 0, (g->e_part + 8) * 4, g->stream));
    if (g->e_part) LUXB_CUDA(cudaMemcpyAsync(g->d_weight, weight_slice, g->e_part * 4, cudaMemcpyDefault, g->stream));
  }
  // every source id of this rank's slice must be a vertex (checked where the data already is: on the device)
  unsigned long long* d_bad = reinterpret_cast<unsigned long long*>(d_tmp);
  LUXB_CUDA(cudaMemsetAsync(d_bad, 0, 8, g->stream));
  if (g->e_part) src_out_of_range_kernel<<<g->num_sms * 8, 256, 0, g->stream>>>(g->d_src, g->e_part, g->nv, d_bad);
  unsigned long long bad = 0;
  LUXB_CUDA(cudaMemcpyAsync(&bad, d_bad, 8, cudaMemcpyDeviceToHost, g->stream));
  LUXB_CUDA(cudaStreamSynchronize(g->stream));
  unsigned long long neg = 0;
  const bool bc = g->cfg.app == LUXB_BC_WEIGHTED;
  if (app_of(g).dist_labels && g->e_part) {  // shortest paths need w >= 0, BC w >= 1 (checked the same way, on the device)
    LUXB_CUDA(cudaMemsetAsync(d_bad, 0, 8, g->stream));
    if (bc) light_weight_kernel<<<g->num_sms * 8, 256, 0, g->stream>>>(g->d_weight, g->e_part, 1, d_bad);
    else negative_weight_kernel<<<g->num_sms * 8, 256, 0, g->stream>>>(g->d_weight, g->e_part, d_bad);
    LUXB_CUDA(cudaMemcpyAsync(&neg, d_bad, 8, cudaMemcpyDeviceToHost, g->stream));
    LUXB_CUDA(cudaStreamSynchronize(g->stream));
  }
  tmp.release(d_tmp);
  LUXB_ARG(bad == 0, "%llu source ids of this rank's slice are >= nv (%u)", bad, g->nv);
  LUXB_ARG(neg == 0 || bc, "%llu edge weights of this rank's slice are negative (weighted SSSP needs w >= 0)", neg);
  LUXB_ARG(neg == 0, "%llu edge weights of this rank's slice are < 1 (weighted betweenness centrality needs w >= 1)", neg);
  return finish_layout(g);
}

// ------------------------------------------------------------------------------------------------------------
extern "C" {

const char* luxb_last_error(void) { return g_err; }
const char* luxb_version(void) { return "lux_b200 0.2 (sm_90a)"; }
int luxb_abi_version(void) { return 3; }

int luxb_partition_csc(luxb_vid nv, luxb_eid ne, const luxb_eid* row_end, int P, luxb_vid* row_left, luxb_vid* row_right,
                       luxb_eid* col_left) {
  LUXB_ARG(row_end && row_left && row_right && col_left, "NULL argument");
  LUXB_ARG(P >= 1 && P <= LUXB_MAX_PARTS, "P out of range");
  LUXB_TRY(validate_row_end(nv, ne, row_end));
  uint32_t np[LUXB_MAX_PARTS];
  int found = host_partition(nv, ne, row_end, P, row_left, np, col_left);
  for (int p = 0; p < P; ++p) row_right[p] = row_left[p] + np[p] - 1;  // empty: row_left - 1
  return found;
}

int luxb_open_csc(const luxb_csc* csc, const luxb_config* cfg, luxb_graph** out) {
  LUXB_ARG(csc && csc->row_end && (csc->src || csc->ne == 0), "csc arrays are NULL");
  LUXB_TRY(check_config(cfg));
  // col_filter needs the weights even without edges (EDGE_WEIGHT, col_filter/app.h:22)
  const AppInfo& app = kApps[cfg->app];
  LUXB_ARG(!app.weights || csc->weight || (csc->ne == 0 && app.dist_labels), "%s needs edge weights", app.name);
  LUXB_TRY(validate_row_end(csc->nv, csc->ne, csc->row_end));
  luxb_graph* g = nullptr;
  int rc = open_host_begin(cfg, csc->nv, csc->ne, csc->row_end, &g);
  if (rc) { if (g) luxb_close(g); return rc; }
  rc = upload_slice(g, csc->row_end + (g->n_part ? g->row_left : 0), csc->src + g->col_left,
                    g->weighted ? csc->weight + g->col_left : nullptr);
  if (rc) { luxb_close(g); return rc; }
  *out = g;
  return 0;
}

int luxb_open_file(const char* path, const luxb_config* cfg, luxb_graph** out) {
  LUXB_ARG(path != nullptr, "path is NULL");
  LUXB_TRY(check_config(cfg));
  FILE* f = fopen(path, "rb");
  if (!f) { set_error("cannot open %s", path); return LUXB_ERR_IO; }
  uint32_t nv = 0;
  uint64_t ne = 0;
  if (fread(&nv, 4, 1, f) != 1 || fread(&ne, 8, 1, f) != 1 || nv == 0) {  // FILE_HEADER_SIZE, core/graph.h:32
    fclose(f);
    set_error("%s: bad .lux header", path);
    return LUXB_ERR_IO;
  }
  std::vector<uint64_t> row_end(nv);
  if (fread(row_end.data(), 8, nv, f) != nv) { fclose(f); set_error("%s: truncated row_end", path); return LUXB_ERR_IO; }
  int rc = validate_row_end(nv, ne, row_end.data());
  if (rc) { fclose(f); return rc; }
  luxb_graph* g = nullptr;
  rc = open_host_begin(cfg, nv, ne, row_end.data(), &g);
  if (rc) { fclose(f); if (g) luxb_close(g); return rc; }
  // this rank's slice only — same seeks as pull_load_task_impl (pull_model.inl:294-318)
  std::vector<uint32_t> src(g->e_part ? g->e_part : 1);
  std::vector<int32_t> w(g->weighted && g->e_part ? g->e_part : 1);
  bool ok = fseeko(f, (off_t)(12 + 8 * (uint64_t)nv + 4 * g->col_left), SEEK_SET) == 0 &&
            fread(src.data(), 4, g->e_part, f) == g->e_part;
  if (ok && g->weighted)
    ok = fseeko(f, (off_t)(12 + 8 * (uint64_t)nv + 4 * ne + 4 * g->col_left), SEEK_SET) == 0 &&
         fread(w.data(), 4, g->e_part, f) == g->e_part;
  fclose(f);
  if (!ok) { luxb_close(g); set_error("%s: truncated edge data", path); return LUXB_ERR_IO; }
  rc = upload_slice(g, row_end.data() + (g->n_part ? g->row_left : 0), src.data(), g->weighted ? w.data() : nullptr);
  if (rc) { luxb_close(g); return rc; }
  *out = g;
  return 0;
}

// ---- .lux writer and edge-list converter (tools/converter.cc) — host only, no device needed -----------------------
int luxb_write_lux(const char* path, const luxb_csc* csc) {
  LUXB_ARG(path && csc && csc->row_end && (csc->src || csc->ne == 0), "NULL argument");
  LUXB_TRY(validate_row_end(csc->nv, csc->ne, csc->row_end));
  std::vector<uint32_t> deg;
  if (!csc->weight) {  // the trailer the reference converter writes: out-degrees (converter.cc:124)
    deg.assign(csc->nv, 0);
    for (uint64_t e = 0; e < csc->ne; ++e) {
      LUXB_ARG(csc->src[e] < csc->nv, "src[%llu] out of range", (unsigned long long)e);
      deg[csc->src[e]]++;
    }
  }
  FILE* f = fopen(path, "wb");
  if (!f) { set_error("cannot create %s", path); return LUXB_ERR_IO; }
  bool ok = fwrite(&csc->nv, 4, 1, f) == 1 && fwrite(&csc->ne, 8, 1, f) == 1 &&       // converter.cc:108-109
            fwrite(csc->row_end, 8, csc->nv, f) == csc->nv &&                          // :110
            (csc->ne == 0 || fwrite(csc->src, 4, csc->ne, f) == csc->ne);              // :112-123
  if (ok && csc->weight) ok = csc->ne == 0 || fwrite(csc->weight, 4, csc->ne, f) == csc->ne;  // EDGE_WEIGHT apps read i32 weights here
  if (ok && !csc->weight) ok = fwrite(deg.data(), 4, csc->nv, f) == csc->nv;                  // :124
  ok = fclose(f) == 0 && ok;
  if (!ok) { set_error("short write to %s", path); return LUXB_ERR_IO; }
  return 0;
}

int luxb_convert_edgelist(const char* edge_list_path, const char* lux_path, luxb_vid nv, luxb_eid ne) {
  LUXB_ARG(edge_list_path && lux_path, "NULL argument");
  LUXB_ARG(nv >= 1, "-nv must be positive");
  FILE* fin = fopen(edge_list_path, "r");
  if (!fin) { set_error("cannot open %s", edge_list_path); return LUXB_ERR_IO; }
  std::vector<uint64_t> keys;  // dst << 32 | src: ascending = canonical (dst, src) order (the reference's std::sort by dst
  keys.reserve(ne);            // leaves the order inside a destination unspecified; ours is deterministic)
  for (uint64_t e = 0; e < ne; ++e) {
    long long a = -1, b = -1;
    if (fscanf(fin, "%lli %lli", &a, &b) != 2) {  // "%i %i" in converter.cc:90: C integer syntax, whitespace separated
      fclose(fin);
      set_error("%s: edge %llu of %llu cannot be read", edge_list_path, (unsigned long long)e, (unsigned long long)ne);
      return LUXB_ERR_IO;
    }
    if (a < 0 || b < 0 || (unsigned long long)a >= nv || (unsigned long long)b >= nv) {  // converter.cc:91-92 asserts
      fclose(fin);
      set_error("%s: edge %llu (%lld -> %lld) has an endpoint outside [0, %u)", edge_list_path, (unsigned long long)e, a, b, nv);
      return LUXB_ERR_ARG;
    }
    keys.push_back(((uint64_t)b << 32) | (uint64_t)a);
  }
  fclose(fin);
  std::sort(keys.begin(), keys.end());
  std::vector<uint64_t> row_end(nv);
  std::vector<uint32_t> src(ne ? ne : 1);
  uint64_t cnt = 0;
  for (uint32_t v = 0; v < nv; ++v) {
    while (cnt < ne && (uint32_t)(keys[cnt] >> 32) == v) { src[cnt] = (uint32_t)keys[cnt]; ++cnt; }
    row_end[v] = cnt;  // END offset of v's in-edge block (converter.cc:100-106)
  }
  luxb_csc csc{nv, ne, row_end.data(), src.data(), nullptr};
  return luxb_write_lux(lux_path, &csc);
}

// a generated graph (GenSpec): partition table and this rank's slice, built on the device
static int generate_slice(luxb_graph* g, const GenSpec& spec) {
  DevTmp tmp;
  const int gen_grid = g->num_sms * 16;
  // 1. in-degree histogram over the whole edge stream -> global row_end (u64) by an inclusive scan
  uint32_t* d_indeg = nullptr;
  uint64_t* d_row_end_g = nullptr;
  LUXB_TRY(tmp.alloc(&d_indeg, spec.nv));
  LUXB_TRY(tmp.alloc(&d_row_end_g, spec.nv));
  LUXB_CUDA(cudaMemsetAsync(d_indeg, 0, (size_t)spec.nv * 4, g->stream));
  gen_count_indeg_kernel<<<gen_grid, 256, 0, g->stream>>>(spec, d_indeg);
  widen_u32_to_u64_kernel<<<gen_grid, 256, 0, g->stream>>>(d_indeg, d_row_end_g, spec.nv);
  LUXB_TRY(cub_call(tmp, g->stream, [&](void* t, size_t& b) {
    return cub::DeviceScan::InclusiveSum(t, b, d_row_end_g, d_row_end_g, (int)spec.nv, g->stream);
  }));
  // 2. partition table (reference greedy split), on the device
  uint32_t* d_pt = nullptr;  // rl[P], np[P]
  uint64_t* d_cl = nullptr;
  int* d_cnt = nullptr;
  LUXB_TRY(tmp.alloc(&d_pt, 2 * LUXB_MAX_PARTS));
  LUXB_TRY(tmp.alloc(&d_cl, LUXB_MAX_PARTS));
  LUXB_TRY(tmp.alloc(&d_cnt, 1));
  partition_kernel<<<1, 1, 0, g->stream>>>(d_row_end_g, spec.nv, spec.ne, g->P, d_pt, d_pt + LUXB_MAX_PARTS, d_cl, d_cnt);
  LUXB_CUDA(cudaMemcpyAsync(g->ref_rl, d_pt, g->P * 4, cudaMemcpyDeviceToHost, g->stream));
  LUXB_CUDA(cudaMemcpyAsync(g->ref_np, d_pt + LUXB_MAX_PARTS, g->P * 4, cudaMemcpyDeviceToHost, g->stream));
  LUXB_CUDA(cudaMemcpyAsync(g->ref_cl, d_cl, g->P * 8, cudaMemcpyDeviceToHost, g->stream));
  LUXB_CUDA(cudaMemcpyAsync(&g->parts_found, d_cnt, 4, cudaMemcpyDeviceToHost, g->stream));
  LUXB_CUDA(cudaStreamSynchronize(g->stream));
  if (use_balanced_split(&g->cfg)) {
    // cost prefix over all vertices (in place of the in-degree scratch), then P - 1 binary searches for the cut points
    uint64_t* d_cost = nullptr;
    LUXB_TRY(tmp.alloc(&d_cost, (uint64_t)spec.nv + 1));
    vertex_cost_kernel<<<gen_grid, 256, 0, g->stream>>>(d_row_end_g, spec.nv, kBalanceHubIndeg, d_cost);
    LUXB_TRY(cub_call(tmp, g->stream, [&](void* t, size_t& b) {
      return cub::DeviceScan::InclusiveSum(t, b, d_cost, d_cost, (int)spec.nv, g->stream);
    }));
    balanced_cut_kernel<<<1, 1, 0, g->stream>>>(d_cost, d_row_end_g, spec.nv, spec.ne, g->P, d_pt, d_pt + LUXB_MAX_PARTS, d_cl);
    LUXB_CUDA(cudaMemcpyAsync(g->rl, d_pt, g->P * 4, cudaMemcpyDeviceToHost, g->stream));
    LUXB_CUDA(cudaMemcpyAsync(g->np, d_pt + LUXB_MAX_PARTS, g->P * 4, cudaMemcpyDeviceToHost, g->stream));
    LUXB_CUDA(cudaMemcpyAsync(g->cl, d_cl, g->P * 8, cudaMemcpyDeviceToHost, g->stream));
    LUXB_CUDA(cudaStreamSynchronize(g->stream));
    tmp.release(d_cost);
  } else {
    use_reference_split(g);
  }
  set_partition_derived(g);
  // 3. local row_end (relative + sentinels)
  LUXB_TRY(gmalloc(g, &g->d_row_end, (uint64_t)g->n_part + 4));
  rowend_rel_kernel<<<grid_for((uint64_t)g->n_part + 4, 256, 4096), 256, 0, g->stream>>>(d_row_end_g, g->row_left, g->n_part,
                                                                                        g->col_left, g->d_row_end);
  LUXB_CUDA(cudaGetLastError());
  LUXB_CUDA(cudaStreamSynchronize(g->stream));
  for (void* q : {(void*)d_indeg, (void*)d_row_end_g, (void*)d_pt, (void*)d_cl, (void*)d_cnt}) tmp.release(q);
  // 4. this partition's edges: regenerate the stream, keep keys (dst_local << 32 | src), radix sort -> canonical CSC
  uint64_t *d_keys = nullptr, *d_keys_alt = nullptr;
  unsigned long long* d_cursor = nullptr;
  LUXB_TRY(tmp.alloc(&d_keys, g->e_part));
  LUXB_TRY(tmp.alloc(&d_keys_alt, g->e_part));
  LUXB_TRY(tmp.alloc(&d_cursor, 1));
  LUXB_CUDA(cudaMemsetAsync(d_cursor, 0, 8, g->stream));
  gen_emit_keys_kernel<<<gen_grid, 256, 0, g->stream>>>(spec, g->row_left, g->n_part, d_cursor, d_keys, g->e_part);
  LUXB_CUDA(cudaGetLastError());
  unsigned long long emitted = 0;
  LUXB_CUDA(cudaMemcpyAsync(&emitted, d_cursor, 8, cudaMemcpyDeviceToHost, g->stream));
  LUXB_CUDA(cudaStreamSynchronize(g->stream));
  if (emitted != g->e_part) {
    set_error("generator emitted %llu edges for this partition, expected %llu", emitted, (unsigned long long)g->e_part);
    return LUXB_ERR_STATE;
  }
  int pbits = 1;
  while ((1ull << pbits) < (uint64_t)g->n_part + 1) ++pbits;
  cub::DoubleBuffer<uint64_t> keys(d_keys, d_keys_alt);
  LUXB_TRY(cub_call(tmp, g->stream, [&](void* t, size_t& b) {
    return cub::DeviceRadixSort::SortKeys(t, b, keys, (long long)g->e_part, 0, 32 + pbits, g->stream);
  }));
  LUXB_TRY(edge_alloc(g, &g->d_src, g->e_part + 8));
  LUXB_CUDA(cudaMemsetAsync(g->d_src, 0, (g->e_part + 8) * 4, g->stream));
  if (g->weighted) {
    LUXB_TRY(edge_alloc(g, &g->d_weight, g->e_part + 8));
    LUXB_CUDA(cudaMemsetAsync(g->d_weight, 0, (g->e_part + 8) * 4, g->stream));
  }
  // bipartite: the ratings 1..5 of the (user, item) pair; RMAT (weighted SSSP): directed weights 1..255
  keys_to_src_kernel<<<gen_grid, 256, 0, g->stream>>>(keys.Current(), g->e_part, g->d_src, spec.kind == 0 ? nullptr : g->d_weight,
                                                      spec.seed, g->row_left);
  if (spec.kind == 0 && g->weighted)
    keys_to_rmat_weight_kernel<<<gen_grid, 256, 0, g->stream>>>(keys.Current(), g->e_part, g->d_weight, spec.seed, g->row_left);
  LUXB_CUDA(cudaGetLastError());
  LUXB_CUDA(cudaStreamSynchronize(g->stream));
  for (void* q : {(void*)d_keys, (void*)d_keys_alt, (void*)d_cursor}) tmp.release(q);
  return finish_layout(g);
}

static int open_generated(const GenSpec& spec, const luxb_config* cfg, luxb_graph** out) {
  luxb_graph* g = nullptr;
  int rc = graph_begin(cfg, spec.nv, spec.ne, &g);
  if (!rc) rc = generate_slice(g, spec);
  if (rc) { if (g) luxb_close(g); return rc; }
  *out = g;
  return 0;
}

int luxb_open_rmat(int scale, luxb_vid nv, luxb_eid ne, uint64_t seed, const luxb_config* cfg, luxb_graph** out) {
  LUXB_TRY(check_config(cfg));
  LUXB_ARG(scale >= 1 && scale <= 31, "scale out of range");
  LUXB_ARG(nv >= 1 && (uint64_t)nv <= (1ull << scale) && nv < 0x7FFFFFFFu, "nv must be in [1, min(2^scale, 2^31 - 2)]");
  LUXB_ARG(cfg->app != LUXB_COLFILTER, "use luxb_open_bipartite for col_filter");
  GenSpec s{};
  s.kind = 0; s.scale = scale; s.nv = nv; s.ne = ne; s.seed = seed;
  return open_generated(s, cfg, out);
}

int luxb_open_bipartite(luxb_vid users, luxb_vid items, luxb_eid ratings, uint64_t seed, const luxb_config* cfg,
                        luxb_graph** out) {
  LUXB_TRY(check_config(cfg));
  LUXB_ARG(users >= 1 && items >= 1, "users and items must be positive");
  LUXB_ARG((uint64_t)users + items < 0x7FFFFFFEull, "users + items must stay below 2^31 - 2");
  GenSpec s{};
  s.kind = 1; s.nv = users + items; s.ne = 2 * ratings; s.seed = seed; s.users = users; s.items = items;
  return open_generated(s, cfg, out);
}

int luxb_graph_info(const luxb_graph* g, luxb_vid* nv, luxb_eid* ne, int* nranks) {
  LUXB_ARG(g != nullptr, "graph is NULL");
  if (nv) *nv = g->nv;
  if (ne) *ne = g->ne;
  if (nranks) *nranks = g->P;
  return 0;
}

int luxb_partition_bounds(const luxb_graph* g, luxb_vid* row_left, luxb_vid* row_right, luxb_eid* col_left,
                          uint64_t* fq_left, uint64_t* fq_right) {
  LUXB_ARG(g != nullptr, "graph is NULL");
  uint64_t fsize = 0;
  for (int p = 0; p < g->P; ++p) {  // always the reference's split (Graph::Graph, pull_model.inl:108-131)
    if (row_left) row_left[p] = g->ref_rl[p];
    if (row_right) row_right[p] = g->ref_rl[p] + g->ref_np[p] - 1;
    if (col_left) col_left[p] = g->ref_cl[p];
    const uint32_t span = g->ref_np[p] ? g->ref_np[p] - 1 : 0;
    uint64_t bytes = 8 + (uint64_t)(span / 16 + 100) * 4;  // sizeof(FrontierHeader) + mySlots * sizeof(V_ID), push_model.inl:393
    if (fq_left) fq_left[p] = fsize;
    fsize += bytes;
    if (fq_right) fq_right[p] = fsize - 1;
  }
  return g->parts_found;
}

int luxb_work_bounds(const luxb_graph* g, luxb_vid* row_left, luxb_vid* row_right, luxb_eid* col_left) {
  LUXB_ARG(g != nullptr, "graph is NULL");
  for (int p = 0; p < g->P; ++p) {
    if (row_left) row_left[p] = g->rl[p];
    if (row_right) row_right[p] = g->rl[p] + g->np[p] - 1;
    if (col_left) col_left[p] = g->cl[p];
  }
  return use_balanced_split(&g->cfg) ? 1 : 0;
}

// ---- communicator ------------------------------------------------------------------------------------------
int luxb_comm_unique_id(char id[LUXB_UNIQUE_ID_BYTES]) {
  LUXB_ARG(id != nullptr, "id is NULL");
  const char* err = nccl().load();
  if (err) { set_error("%s", err); return LUXB_ERR_COMM; }
  ncclUniqueId uid;
  LUXB_NCCL(nccl().GetUniqueId(&uid));
  memcpy(id, &uid, LUXB_UNIQUE_ID_BYTES);
  return 0;
}

int luxb_comm_init(luxb_graph* g, const char id[LUXB_UNIQUE_ID_BYTES]) {
  LUXB_ARG(g != nullptr, "graph is NULL");
  if (g->P == 1) return 0;
  LUXB_ARG(id != nullptr, "id is NULL");
  LUXB_ARG(g->comm == nullptr, "communicator already initialised");
  const char* err = nccl().load();
  if (err) { set_error("%s", err); return LUXB_ERR_COMM; }
  LUXB_CUDA(cudaSetDevice(g->cfg.device));
  ncclUniqueId uid;
  memcpy(&uid, id, LUXB_UNIQUE_ID_BYTES);
  LUXB_NCCL(nccl().CommInitRank(&g->comm, g->P, uid, g->cfg.rank));
  // second stream: the cold half of the PageRank exchange overlaps with the next sweep's panel kernel
  LUXB_CUDA(cudaStreamCreateWithFlags(&g->stream2, cudaStreamNonBlocking));
  LUXB_CUDA(cudaEventCreateWithFlags(&g->ev_pack, cudaEventDisableTiming));
  LUXB_CUDA(cudaEventCreateWithFlags(&g->ev_cold, cudaEventDisableTiming));
  return 0;
}

struct P2PBlob {
  cudaIpcMemHandle_t val[2];  // natural-order replicas (col_filter stores into its peers' replicas)
  cudaIpcMemHandle_t xt[2];   // PageRank: packed transfer arrays
  cudaIpcMemHandle_t fq;      // CC / SSSP: frontier slots of every partition (val[0] = label replica)
  cudaIpcMemHandle_t flags;   // barrier flag words (flag_barrier_kernel)
  int has_val, has_xt, has_fq, has_flags;
};

int luxb_p2p_export(luxb_graph* g, void* blob, size_t* blob_bytes) {
  LUXB_ARG(g && blob_bytes, "NULL argument");
  if (!blob) { *blob_bytes = sizeof(P2PBlob); return 0; }
  LUXB_ARG(*blob_bytes >= sizeof(P2PBlob), "blob too small");
  if (!g->inited) { set_error("luxb_p2p_export: call luxb_init first"); return LUXB_ERR_STATE; }
  P2PBlob b;
  memset(&b, 0, sizeof(b));
  LUXB_CUDA(cudaSetDevice(g->cfg.device));
  if (g->cfg.app != LUXB_PAGERANK) {
    for (int k = 0; k < 2; ++k)
      if (g->d_val[k]) LUXB_CUDA(cudaIpcGetMemHandle(&b.val[k], g->d_val[k]));
    b.has_val = 1;
  }
  if (g->d_fq_all) { LUXB_CUDA(cudaIpcGetMemHandle(&b.fq, g->d_fq_all)); b.has_fq = 1; }
  if (g->packed) {
    for (int k = 0; k < 2; ++k) LUXB_CUDA(cudaIpcGetMemHandle(&b.xt[k], g->d_xt[k]));
    b.has_xt = 1;
  }
  if (g->flag_barrier) {
    if (!g->d_flags) {
      LUXB_TRY(gmalloc(g, &g->d_flags, LUXB_MAX_PARTS));
      LUXB_CUDA(cudaMemset(g->d_flags, 0, sizeof(uint32_t) * LUXB_MAX_PARTS));  // before any peer can learn the handle
      LUXB_TRY(gmalloc(g, &g->h_barrier_err, 1, MemKind::kMapped));
      *g->h_barrier_err = 0;
    }
    LUXB_CUDA(cudaIpcGetMemHandle(&b.flags, g->d_flags));
    b.has_flags = 1;
  }
  memcpy(blob, &b, sizeof(b));
  *blob_bytes = sizeof(P2PBlob);
  return 0;
}

static void p2p_unmap(luxb_graph* g);

int luxb_p2p_import(luxb_graph* g, const void* all_blobs, size_t blob_bytes_each) {
  LUXB_ARG(g && all_blobs, "NULL argument");
  LUXB_ARG(blob_bytes_each == sizeof(P2PBlob), "blob size mismatch");
  if (!g->inited) { set_error("luxb_p2p_import: call luxb_init first"); return LUXB_ERR_STATE; }
  if (g->P == 1) return 0;
  LUXB_ARG(g->comm != nullptr, "P2P exchange still needs the communicator for its iteration barrier");
  LUXB_CUDA(cudaSetDevice(g->cfg.device));
  const P2PBlob* blobs = reinterpret_cast<const P2PBlob*>(all_blobs);
  // an import that fails half-way leaves nothing mapped (p2p_unmap)
  bool all_flags = g->flag_barrier && g->d_flags;
  for (int p = 0; p < g->P; ++p) all_flags = all_flags && (p == g->cfg.rank || blobs[p].has_flags);
  for (int p = 0; p < g->P; ++p) {
    if (p == g->cfg.rank) {
      for (int k = 0; k < 2; ++k) { g->peer_val[k][p] = g->d_val[k]; g->peer_xt[k][p] = g->d_xt[k]; }
      g->peer_fq[p] = g->d_fq_all;
      g->peer_flags[p] = g->d_flags;
      continue;
    }
    if (all_flags) {
      cudaError_t e = cudaIpcOpenMemHandle(&g->peer_flags[p], blobs[p].flags, cudaIpcMemLazyEnablePeerAccess);
      if (e != cudaSuccess) {
        set_error("cudaIpcOpenMemHandle (rank %d's barrier flags): %s", p, cudaGetErrorString(e));
        p2p_unmap(g);
        return LUXB_ERR_CUDA;
      }
    }
    if (blobs[p].has_fq && g->d_fq_all) {
      cudaError_t e = cudaIpcOpenMemHandle(&g->peer_fq[p], blobs[p].fq, cudaIpcMemLazyEnablePeerAccess);
      if (e != cudaSuccess) {
        set_error("cudaIpcOpenMemHandle (rank %d's frontier slots): %s", p, cudaGetErrorString(e));
        p2p_unmap(g);
        return LUXB_ERR_CUDA;
      }
    }
    for (int k = 0; k < 2; ++k) {
      cudaError_t e = cudaSuccess;
      if (blobs[p].has_val && g->d_val[k]) e = cudaIpcOpenMemHandle(&g->peer_val[k][p], blobs[p].val[k], cudaIpcMemLazyEnablePeerAccess);
      if (e == cudaSuccess && blobs[p].has_xt && g->d_xt[k])
        e = cudaIpcOpenMemHandle(&g->peer_xt[k][p], blobs[p].xt[k], cudaIpcMemLazyEnablePeerAccess);
      if (e != cudaSuccess) {
        set_error("cudaIpcOpenMemHandle (rank %d's buffers): %s", p, cudaGetErrorString(e));
        p2p_unmap(g);
        return LUXB_ERR_CUDA;
      }
    }
  }
  g->flag_barrier = all_flags;  // every rank decides alike: the blobs are the same everywhere
  g->p2p_ready = true;
  return 0;
}

int luxb_p2p_disable(luxb_graph* g) {
  LUXB_ARG(g != nullptr, "graph is NULL");
  g->p2p_ready = false;
  return 0;
}

// close every peer buffer mapped into this process
static void p2p_unmap(luxb_graph* g) {
  for (int p = 0; p < g->P; ++p) {
    if (p == g->cfg.rank) continue;
    for (int k = 0; k < 2; ++k) {
      if (g->peer_val[k][p]) { cudaIpcCloseMemHandle(g->peer_val[k][p]); g->peer_val[k][p] = nullptr; }
      if (g->peer_xt[k][p]) { cudaIpcCloseMemHandle(g->peer_xt[k][p]); g->peer_xt[k][p] = nullptr; }
    }
    if (g->peer_fq[p]) { cudaIpcCloseMemHandle(g->peer_fq[p]); g->peer_fq[p] = nullptr; }
    if (g->peer_flags[p]) { cudaIpcCloseMemHandle(g->peer_flags[p]); g->peer_flags[p] = nullptr; }
  }
  g->p2p_ready = false;
}

int luxb_p2p_disconnect(luxb_graph* g) {
  LUXB_ARG(g != nullptr, "graph is NULL");
  LUXB_CUDA(cudaSetDevice(g->cfg.device));
  if (g->stream) LUXB_CUDA(cudaStreamSynchronize(g->stream));
  if (g->stream2) LUXB_CUDA(cudaStreamSynchronize(g->stream2));  // a cold pull may still be reading the peers' transfer arrays
  p2p_unmap(g);
  return 0;
}

// ---- init ---------------------------------------------------------------------------------------------------
static int build_push_csr(luxb_graph* g) {
  // CSR-by-source over this partition's own edges (init_push_* kernels, components_gpu.cu:550-607):
  // stable radix sort of (src, dst) pairs by src keeps each source's destinations ascending -> deterministic.
  DevTmp tmp;  // temporaries are released on every exit path
  LUXB_TRY(gmalloc(g, &g->d_out_end, g->nv));
  LUXB_TRY(gmalloc(g, &g->d_out_dst, g->e_part));
  uint32_t* d_cnt = nullptr;
  LUXB_TRY(tmp.alloc(&d_cnt, g->nv));
  LUXB_CUDA(cudaMemsetAsync(d_cnt, 0, (size_t)g->nv * 4, g->stream));
  const int grid = g->num_sms * 8;
  hist_src_kernel<<<grid, 256, 0, g->stream>>>(g->d_src, g->e_part, d_cnt);
  widen_u32_to_u64_kernel<<<grid, 256, 0, g->stream>>>(d_cnt, g->d_out_end, g->nv);
  LUXB_TRY(cub_call(tmp, g->stream, [&](void* t, size_t& b) {
    return cub::DeviceScan::InclusiveSum(t, b, g->d_out_end, g->d_out_end, (int)g->nv, g->stream);
  }));
  tmp.release(d_cnt);
  if (g->e_part == 0) return 0;
  uint32_t *d_dst = nullptr, *d_keys_out = nullptr;
  LUXB_TRY(tmp.alloc(&d_dst, g->e_part));
  LUXB_TRY(tmp.alloc(&d_keys_out, g->e_part));
  edge_dst_kernel<<<grid, 256, 0, g->stream>>>(g->d_row_end, g->n_part, g->e_part, g->row_left, d_dst);
  LUXB_CUDA(cudaGetLastError());
  int vbits = 1;
  while ((1ull << vbits) < (uint64_t)g->nv) ++vbits;
  LUXB_TRY(cub_call(tmp, g->stream, [&](void* t, size_t& b) {
    return cub::DeviceRadixSort::SortPairs(t, b, g->d_src, d_keys_out, d_dst, g->d_out_dst, (long long)g->e_part, 0, vbits, g->stream);
  }));
  if (app_of(g).dist_labels) {
    // the weights in the same order: the same stable sort on the same keys applies the same permutation
    LUXB_TRY(gmalloc(g, &g->d_out_w, g->e_part));
    LUXB_TRY(cub_call(tmp, g->stream, [&](void* t, size_t& b) {
      return cub::DeviceRadixSort::SortPairs(t, b, g->d_src, d_keys_out, g->d_weight, g->d_out_w, (long long)g->e_part, 0, vbits,
                                             g->stream);
    }));
  }
  return 0;
}

static unsigned char* slot_ptr(unsigned char* base, const luxb_graph* g, int p) { return base + g->slot_off[p]; }

// initial labels + frontier (components_gpu.cu:733-739; sssp_gpu.cu:733-744) — every rank builds all slots locally.
// `start`: the SSSP start vertex (cfg.start_vtx, or the current source of betweenness centrality)
static int reset_label_state(luxb_graph* g, bool all_active, uint32_t start) {
  const bool cc = g->cfg.app == LUXB_CC;
  uint32_t* lab = reinterpret_cast<uint32_t*>(g->d_val[0]);
  LUXB_CUDA(cudaMemsetAsync(g->d_fq_all, 0, g->fq_total, g->stream));
  for (int p = 0; p < g->P; ++p) {
    FrontierHeader h;
    unsigned char* slot = slot_ptr(g->d_fq_all, g, p);
    if (cc || all_active) {
      h.type = LUXB_DENSE_BITMAP;
      h.num_nodes = g->np[p];
      uint64_t bytes = g->np[p] ? (g->np[p] - 1) / 8 + 1 : 0;  // (R-L)/8 + 1, components_gpu.cu:737
      if (bytes) LUXB_CUDA(cudaMemsetAsync(slot + 8, 0xFF, bytes, g->stream));
    } else {
      h.type = LUXB_SPARSE_QUEUE;
      bool mine = g->np[p] && start >= g->rl[p] && start - g->rl[p] < g->np[p];
      h.num_nodes = mine ? 1 : 0;
      if (mine) {
        uint32_t q[1] = {start};
        uint32_t zero[1] = {0};
        LUXB_CUDA(cudaMemcpyAsync(slot + 8, q, 4, cudaMemcpyHostToDevice, g->stream));
        LUXB_CUDA(cudaMemcpyAsync(slot + 8 + (size_t)g->cap[p] * 4, zero, 4, cudaMemcpyHostToDevice, g->stream));
      }
    }
    LUXB_CUDA(cudaMemcpyAsync(slot, &h, 8, cudaMemcpyHostToDevice, g->stream));
    g->h_hdr[2 * p] = h.type;
    g->h_hdr[2 * p + 1] = h.num_nodes;
  }
  if (!all_active) {
    const int grid = g->num_sms * 8;
    if (cc) iota_kernel<<<grid, 256, 0, g->stream>>>(lab, g->nv);
    else {
      // INF: nv for hop counts (sssp_gpu.cu:733-744), LUXB_DIST_INF for weighted distances
      fill_kernel<uint32_t><<<grid, 256, 0, g->stream>>>(lab, g->nv, app_of(g).dist_labels ? kDistInf : g->nv);
      uint32_t zero = 0;
      if (start < g->nv)
        LUXB_CUDA(cudaMemcpyAsync(lab + start, &zero, 4, cudaMemcpyHostToDevice, g->stream));
    }
    LUXB_CUDA(cudaGetLastError());
  }
  if (g->n_part)
    LUXB_CUDA(cudaMemcpyAsync(g->d_cur, lab + g->row_left, (size_t)g->n_part * 4, cudaMemcpyDeviceToDevice, g->stream));
  LUXB_CUDA(cudaStreamSynchronize(g->stream));
  g->stats.last_active = 0;
  for (int p = 0; p < g->P; ++p) g->stats.last_active += g->h_hdr[2 * p + 1];
  g->stats.last_frontier_type = g->h_hdr[2 * g->cfg.rank];
  return 0;
}

// Pin the hot copies in L2: persisting access-policy window on the hot buffer for every kernel of this stream,
// everything else is treated as streaming when it misses.  LUXB_L2_PERSIST=0 disables.  With the cold-hub stream the
// window covers only the hottest kColdSplitWindowMB: while that kernel runs, the persisting lines hold values it never
// reads, and L2 is what keeps its cold segment close.
static constexpr double kColdSplitWindowMB = 12.0;
static int set_l2_persisting_window(luxb_graph* g, void* base, size_t bytes) {
  if (!g->sweep.l2_persist) return 0;
  int max_persist = 0, max_window = 0;
  LUXB_CUDA(cudaDeviceGetAttribute(&max_persist, cudaDevAttrMaxPersistingL2CacheSize, g->cfg.device));
  LUXB_CUDA(cudaDeviceGetAttribute(&max_window, cudaDevAttrMaxAccessPolicyWindowSize, g->cfg.device));
  if (max_persist <= 0 || max_window <= 0) return 0;
  if (g->sweep.l2_window_mb >= 0) bytes = std::min<size_t>(bytes, (size_t)(g->sweep.l2_window_mb * 1e6));  // hottest prefix only
  else if (g->cs_on) bytes = std::min<size_t>(bytes, (size_t)(kColdSplitWindowMB * 1e6));
  size_t persist = std::min<size_t>((size_t)max_persist, bytes);
  LUXB_CUDA(cudaDeviceSetLimit(cudaLimitPersistingL2CacheSize, persist));
  cudaStreamAttrValue attr{};
  attr.accessPolicyWindow.base_ptr = base;
  attr.accessPolicyWindow.num_bytes = std::min<size_t>(bytes, (size_t)max_window);
  attr.accessPolicyWindow.hitRatio = (float)std::min(1.0, (double)persist / (double)attr.accessPolicyWindow.num_bytes);
  attr.accessPolicyWindow.hitProp = cudaAccessPropertyPersisting;
  attr.accessPolicyWindow.missProp = cudaAccessPropertyStreaming;
  LUXB_CUDA(cudaStreamSetAttribute(g->stream, cudaStreamAttributeAccessPolicyWindow, &attr));
  if (g->stream_b) LUXB_CUDA(cudaStreamSetAttribute(g->stream_b, cudaStreamAttributeAccessPolicyWindow, &attr));
  if (g->cfg.verbose) printf("L2 persisting window: %zu bytes (device max persisting %d, max window %d)\n", persist, max_persist, max_window);
  return 0;
}

// cold -> hub edges (PageRank, one rank) get a stream of their own when they are at least this share of the partition
static constexpr double kColdSplitMinShare = 0.05;
// the automatic source-blocked split, its tiers and its cold-hub stream only consider partitions of this many edges
static constexpr uint64_t kSplitMinEdges = 1ull << 24;

// May the source-blocked split (build_panel_layout) run on this partition?  It still declines after keying when the
// panel would cover too few edges.
static bool split_may_run(const luxb_graph* g) {
  const SweepSettings& s = g->sweep;
  return s.seg && s.sb != 0 && !g->cfg.zero_copy_edges && (s.sb > 0 || g->e_part >= kSplitMinEdges);
}

// Choose the hot set (largest out-degrees, at most LUXB_HOT_MB megabytes of values, default 24 MB ~ half of the H100's
// 50 MB L2: at RMAT-27 on one H100 8 / 16 / 24 / 32 / 64 MB gave 21.4 / 15.8 / 14.2 / 16.7 / 17.3 ms per sweep) and
// rewrite this partition's source ids as indices into the gather space Z = [hot copies in global hotness order | cold]
// (see build.cuh).  cold = the natural-order value array, or — compact_cold (PageRank) — only the cold vertices that are
// ever gathered, in id order: on several ranks the cold part of the packed exchange, on one rank a copy stored right
// after the hot copies (Z = [hot | cold] in one buffer, refreshed with them by one gather over d_hot_order).
static int build_hot_layout(luxb_graph* g, bool compact_cold) {
  g->hot_n = 0;
  g->packed = false;
  g->cold_z = false;
  uint64_t h_max = (uint64_t)(g->sweep.hot_mb * 1e6 / 4.0);
  if (h_max == 0 || g->nv < 2 || (uint64_t)g->nv >= 0xFFFFFFFFull - h_max) return 0;
  if (h_max > g->nv) h_max = g->nv;
  const int grid = g->num_sms * 8;
  const uint32_t cap = 4096;
  DevTmp tmp;
  unsigned long long* d_hist = nullptr;
  LUXB_TRY(tmp.alloc(&d_hist, cap + 1));
  LUXB_CUDA(cudaMemsetAsync(d_hist, 0, (cap + 1) * 8, g->stream));
  degree_hist_kernel<<<grid, 256, 0, g->stream>>>(g->d_deg, g->nv, cap, d_hist);
  std::vector<unsigned long long> hist(cap + 1);
  LUXB_CUDA(cudaMemcpyAsync(hist.data(), d_hist, (cap + 1) * 8, cudaMemcpyDeviceToHost, g->stream));
  LUXB_CUDA(cudaStreamSynchronize(g->stream));
  // smallest tau >= 2 with |{deg >= tau}| <= h_max  (degree-1 vertices are gathered once: packing cannot help them)
  uint64_t above = 0;
  uint32_t tau = cap + 1;
  for (uint32_t d = cap; d >= 2; --d) {
    if (above + hist[d] > h_max) break;
    above += hist[d];
    tau = d;
  }
  if (above == 0 || tau > cap) return 0;
  const uint32_t H = (uint32_t)above;
  if (compact_cold && g->P == 1) {
    // one rank: the compact cold copy costs a refresh every iteration and pays for it in the cold-hub stream
    // (build_panel_layout).  LUXB_CS = 0: never, 1: always, unset: when the edges out of cold vertices are at least
    // kColdSplitMinShare of a large partition the source-blocked split may sweep (the cold-hub stream needs its hubs)
    const int cs_mode = g->sweep.cs;
    uint64_t e_cold_src = 0;
    for (uint32_t d = 1; d < tau; ++d) e_cold_src += (uint64_t)d * hist[d];
    if (cs_mode == 0 || (cs_mode < 0 && (!split_may_run(g) || g->e_part < kSplitMinEdges ||
                                         (double)e_cold_src < kColdSplitMinShare * (double)g->e_part)))
      compact_cold = false;
  }
  uint64_t *d_keys = nullptr, *d_keys2 = nullptr;
  uint32_t *d_ids = nullptr, *d_ids2 = nullptr, *d_map = nullptr;
  unsigned int* d_cursor = nullptr;  // [0] cursor, [1 .. P] per-owner counts
  LUXB_TRY(tmp.alloc(&d_keys, H));
  LUXB_TRY(tmp.alloc(&d_keys2, H));
  LUXB_TRY(tmp.alloc(&d_ids, H));
  LUXB_TRY(tmp.alloc(&d_ids2, H));
  LUXB_TRY(gmalloc(g, &g->d_hot_order, H));
  LUXB_TRY(tmp.alloc(&d_cursor, 1 + LUXB_MAX_PARTS));
  LUXB_CUDA(cudaMemsetAsync(d_cursor, 0, 4 * (1 + LUXB_MAX_PARTS), g->stream));
  PartTable pt{};
  pt.P = g->P;
  for (int p = 0; p < g->P; ++p) { pt.rl[p] = g->rl[p]; pt.np[p] = g->np[p]; }
  hot_select_kernel<<<grid, 256, 0, g->stream>>>(g->d_deg, g->nv, tau, pt, d_cursor, d_cursor + 1, d_keys, d_ids, H);
  LUXB_CUDA(cudaGetLastError());
  // ids arrive in nondeterministic order: sort by (key, id) = two stable passes (id first, then key)
  int vbits = 1;
  while ((1ull << vbits) < (uint64_t)g->nv) ++vbits;
  LUXB_TRY(cub_call(tmp, g->stream, [&](void* t, size_t& b) {
    return cub::DeviceRadixSort::SortPairs(t, b, d_ids, d_ids2, d_keys, d_keys2, (int)H, 0, vbits, g->stream);
  }));
  LUXB_TRY(cub_call(tmp, g->stream, [&](void* t, size_t& b) {
    return cub::DeviceRadixSort::SortPairs(t, b, d_keys2, d_keys, d_ids2, g->d_hot_order, (int)H, 0, 32, g->stream);
  }));
  unsigned int h_cnt[1 + LUXB_MAX_PARTS];
  LUXB_CUDA(cudaMemcpyAsync(h_cnt, d_cursor, sizeof(h_cnt), cudaMemcpyDeviceToHost, g->stream));
  LUXB_CUDA(cudaStreamSynchronize(g->stream));
  g->hot_off[0] = 0;
  for (int p = 0; p < g->P; ++p) g->hot_off[p + 1] = g->hot_off[p] + h_cnt[1 + p];
  LUXB_TRY(tmp.alloc(&d_map, g->nv));
  uint32_t *d_cflag = nullptr, *d_crank = nullptr;
  if (compact_cold) {
    // cold-active vertices (0 < deg < tau), ranked in id order; owner p's share is [cold_off[p], cold_off[p+1])
    LUXB_TRY(tmp.alloc(&d_cflag, (uint64_t)g->nv + 1));
    LUXB_TRY(tmp.alloc(&d_crank, (uint64_t)g->nv + 1));
    cold_flag_kernel<<<grid, 256, 0, g->stream>>>(g->d_deg, g->nv, tau, d_cflag);
    LUXB_CUDA(cudaMemsetAsync(d_cflag + g->nv, 0, 4, g->stream));
    LUXB_TRY(cub_call(tmp, g->stream, [&](void* t, size_t& b) {
      return cub::DeviceScan::ExclusiveSum(t, b, d_cflag, d_crank, (int)g->nv + 1, g->stream);
    }));
    for (int p = 0; p <= g->P; ++p) {
      const uint32_t at = p < g->P ? std::min(g->rl[p], g->nv) : g->nv;  // empty partitions sit at nv
      LUXB_CUDA(cudaMemcpyAsync(&g->cold_off[p], d_crank + at, 4, cudaMemcpyDeviceToHost, g->stream));
    }
    LUXB_CUDA(cudaStreamSynchronize(g->stream));
    g->cold_n = g->cold_off[g->P];
    gather_map_compact_kernel<<<grid, 256, 0, g->stream>>>(d_map, d_crank, g->nv, H);
  } else {
    gather_map_init_kernel<<<grid, 256, 0, g->stream>>>(d_map, g->nv, H);
  }
  if (compact_cold && g->P == 1) {
    // d_hot_order becomes [hot order | cold-active vertices in id order]: the refresh gather fills all of Z
    uint32_t* d_zsrc = nullptr;
    LUXB_TRY(gmalloc(g, &d_zsrc, (uint64_t)H + g->cold_n + 1));
    LUXB_CUDA(cudaMemcpyAsync(d_zsrc, g->d_hot_order, (size_t)H * 4, cudaMemcpyDeviceToDevice, g->stream));
    pack_list_cold_kernel<<<grid, 256, 0, g->stream>>>(d_cflag, d_crank, 0, g->nv, 0, d_zsrc + H);
    LUXB_CUDA(cudaGetLastError());
    LUXB_CUDA(cudaStreamSynchronize(g->stream));
    LUXB_TRY(gfree(g, g->d_hot_order));
    g->d_hot_order = d_zsrc;
    g->cold_z = true;
  } else if (compact_cold) {
    uint32_t *d_okeys = nullptr, *d_okeys2 = nullptr, *d_ranks = nullptr;
    // transfer order of the hot values: grouped by owner (stable: hotness order inside a group)
    LUXB_TRY(tmp.alloc(&d_okeys, H));
    LUXB_TRY(tmp.alloc(&d_okeys2, H));
    LUXB_TRY(tmp.alloc(&d_ranks, H));
    LUXB_TRY(gmalloc(g, &g->d_zperm, H));
    owner_keys_kernel<<<grid, 256, 0, g->stream>>>(g->d_hot_order, H, pt, d_okeys, d_ranks);
    LUXB_CUDA(cudaGetLastError());
    LUXB_TRY(cub_call(tmp, g->stream, [&](void* t, size_t& b) {
      return cub::DeviceRadixSort::SortPairs(t, b, d_okeys, d_okeys2, d_ranks, g->d_zperm, (int)H, 0, 8, g->stream);
    }));
    const int me = g->cfg.rank;
    const uint32_t nh_me = g->hot_off[me + 1] - g->hot_off[me], nc_me = g->cold_off[me + 1] - g->cold_off[me];
    LUXB_TRY(gmalloc(g, &g->d_pack_list, (uint64_t)nh_me + nc_me + 1));
    if (nh_me)
      pack_list_hot_kernel<<<grid_for(nh_me, 256, grid), 256, 0, g->stream>>>(g->d_hot_order, g->d_zperm, g->hot_off[me], nh_me, g->row_left,
                                                                              g->d_pack_list);
    if (g->n_part)
      pack_list_cold_kernel<<<grid, 256, 0, g->stream>>>(d_cflag, d_crank, g->row_left, g->n_part, g->cold_off[me], g->d_pack_list + nh_me);
    LUXB_CUDA(cudaGetLastError());
    g->packed = true;
  }
  gather_map_hot_kernel<<<grid, 256, 0, g->stream>>>(d_map, g->d_hot_order, H);
  LUXB_TRY(edge_alloc(g, &g->d_src_gather, g->e_part + 8));
  LUXB_CUDA(cudaMemsetAsync(g->d_src_gather, 0, (g->e_part + 8) * 4, g->stream));
  remap_src_kernel<<<grid, 256, 0, g->stream>>>(g->d_src, g->e_part, d_map, g->d_src_gather);
  LUXB_CUDA(cudaGetLastError());
  LUXB_CUDA(cudaStreamSynchronize(g->stream));
  g->hot_n = H;
  return 0;
}

static int allgather_slices(luxb_graph* g, void* replica, size_t elem_bytes);
static void resolve_sweep_settings(SweepSettings& s);
static int build_seg_sweep(luxb_graph* g);
static int pagerank_publish(luxb_graph* g, float* x_new);
static int wait_cold_exchange(luxb_graph* g);
static int bc_alloc(luxb_graph* g);
static int tc_build(luxb_graph* g);
static int kcore_build(luxb_graph* g);
static int truss_build(luxb_graph* g);

// The gather side of the pull sweeps: global out-degrees, the hot set (build_hot_layout), the flagged streams if
// `streams` (build_seg_sweep) and the hot copies Z = [hot | compact cold values on one rank] + one whole table of slack:
// the panel kernel always bulk-loads full blocks (panel.cuh); only the hot prefix gets the persisting window
static int build_gather_side(luxb_graph* g, bool compact_cold, bool streams) {
  LUXB_TRY(gmalloc(g, &g->d_deg, g->nv));
  LUXB_CUDA(cudaMemsetAsync(g->d_deg, 0, (size_t)g->nv * 4, g->stream));
  hist_src_kernel<<<g->num_sms * 8, 256, 0, g->stream>>>(g->d_src, g->e_part, g->d_deg);  // pull_scan_task_impl
  LUXB_CUDA(cudaGetLastError());
  if (g->P > 1) LUXB_NCCL(nccl().AllReduce(g->d_deg, g->d_deg, g->nv, ncclUint32, ncclSum, g->comm, g->stream));
  LUXB_TRY(build_hot_layout(g, compact_cold));
  if (streams) LUXB_TRY(build_seg_sweep(g));
  if (g->sb_on && g->P == 1) {  // the side stream of the concurrent split sweep (sweep_seg)
    LUXB_CUDA(cudaStreamCreateWithFlags(&g->stream_b, cudaStreamNonBlocking));
    LUXB_CUDA(cudaEventCreateWithFlags(&g->ev_fork, cudaEventDisableTiming));
    LUXB_CUDA(cudaEventCreateWithFlags(&g->ev_join, cudaEventDisableTiming));
  }
  if (g->hot_n) {
    const uint64_t z_len = (uint64_t)g->hot_n + (g->cold_z ? g->cold_n : 0) + 65536;
    LUXB_TRY(gmalloc(g, (uint32_t**)&g->d_hot, z_len));
    LUXB_CUDA(cudaMemsetAsync(g->d_hot, 0, z_len * 4, g->stream));
    LUXB_TRY(set_l2_persisting_window(g, g->d_hot, (size_t)g->hot_n * 4));
  }
  return 0;
}

int luxb_init(luxb_graph* g) {
  LUXB_ARG(g != nullptr, "graph is NULL");
  if (g->inited) { set_error("luxb_init called twice"); return LUXB_ERR_STATE; }
  if (g->P > 1 && !g->comm) { set_error("luxb_init: nranks > 1 needs luxb_comm_init first"); return LUXB_ERR_STATE; }
  LUXB_CUDA(cudaSetDevice(g->cfg.device));
  resolve_sweep_settings(g->sweep);
  const int grid = g->num_sms * 8;
  switch (g->cfg.app) {
    case LUXB_PAGERANK: {
      LUXB_TRY(build_gather_side(g, /*compact_cold=*/true, /*streams=*/true));
      for (int k = 0; k < 2; ++k) LUXB_TRY(gmalloc(g, (float**)&g->d_val[k], (uint64_t)g->nv + 64));
      pr_init_kernel<<<grid, 256, 0, g->stream>>>(g->d_deg, g->nv, (float*)g->d_val[0]);
      LUXB_CUDA(cudaMemsetAsync(g->d_val[1], 0, (size_t)g->nv * 4, g->stream));
      if (g->packed) {
        g->xt_hot_chunk = ((((uint64_t)g->hot_n + g->P - 1) / g->P) + 31) & ~31ull;
        g->xt_cold_chunk = ((((uint64_t)g->cold_n + g->P - 1) / g->P) + 31) & ~31ull;
        const uint64_t xt_len = (g->xt_hot_chunk + g->xt_cold_chunk) * g->P;
        for (int k = 0; k < 2; ++k) {
          LUXB_TRY(gmalloc(g, &g->d_xt[k], xt_len));
          LUXB_CUDA(cudaMemsetAsync(g->d_xt[k], 0, xt_len * 4, g->stream));
        }
      }
      LUXB_CUDA(cudaGetLastError());
      // every rank holds the complete x0: publish it (packs this rank's share, exchanges, fills the hot copies)
      LUXB_TRY(pagerank_publish(g, (float*)g->d_val[0]));
      g->replica_stale = false;
      break;
    }
    case LUXB_COLFILTER: {
      for (int k = 0; k < 2; ++k) LUXB_TRY(gmalloc(g, (float**)&g->d_val[k], (uint64_t)g->nv * kCfK));
      cf_init_kernel<<<grid, 256, 0, g->stream>>>((float*)g->d_val[0], (uint64_t)g->nv * kCfK);
      cf_init_kernel<<<grid, 256, 0, g->stream>>>((float*)g->d_val[1], (uint64_t)g->nv * kCfK);
      // chunk table
      DevTmp tmp;
      uint32_t* d_cnt = nullptr;
      LUXB_TRY(tmp.alloc(&d_cnt, (uint64_t)g->n_part + 1));
      LUXB_TRY(gmalloc(g, &g->cf.chunk_first, (uint64_t)g->n_part + 2));
      LUXB_CUDA(cudaMemsetAsync(d_cnt, 0, ((size_t)g->n_part + 1) * 4, g->stream));
      cf_chunk_count_kernel<<<grid, 256, 0, g->stream>>>(g->d_row_end, g->n_part, d_cnt);
      LUXB_TRY(cub_call(tmp, g->stream, [&](void* t, size_t& b) {
        return cub::DeviceScan::ExclusiveSum(t, b, d_cnt, g->cf.chunk_first, (int)g->n_part + 1, g->stream);
      }));
      LUXB_CUDA(cudaMemcpyAsync(&g->cf.n_chunks, g->cf.chunk_first + g->n_part, 4, cudaMemcpyDeviceToHost, g->stream));
      LUXB_CUDA(cudaStreamSynchronize(g->stream));
      tmp.release(d_cnt);
      LUXB_TRY(gmalloc(g, &g->cf.chunk_vtx, g->cf.n_chunks));
      LUXB_TRY(gmalloc(g, &g->cf.partial, (uint64_t)g->cf.n_chunks * kCfK));
      cf_chunk_fill_kernel<<<grid, 256, 0, g->stream>>>(g->cf.chunk_first, g->n_part, g->cf.chunk_vtx);
      LUXB_CUDA(cudaGetLastError());
      break;
    }
    case LUXB_CC:
    case LUXB_SSSP:
    case LUXB_SSSP_WEIGHTED:
    case LUXB_BC:
    case LUXB_BC_WEIGHTED: {  // betweenness centrality: SSSP's state for the search of every source, then its own arrays (bc_alloc)
      LUXB_ARG(app_of(g).run != AppRun::kConvergence || g->cfg.app == LUXB_CC || g->cfg.start_vtx < g->nv, "start vertex %u >= nv",
               g->cfg.start_vtx);
      LUXB_TRY(gmalloc(g, (uint32_t**)&g->d_val[0], g->nv));
      LUXB_TRY(gmalloc(g, &g->d_cur, g->n_part));
      LUXB_TRY(build_push_csr(g));
      // hot-packed label copies for the pull sweeps (same layout as PageRank; refreshed before every pull sweep).
      // Weighted distances are pulled through the merge-path sweep only: the flagged streams carry no weights.
      LUXB_TRY(build_gather_side(g, /*compact_cold=*/false, /*streams=*/!app_of(g).dist_labels));
      g->big_capacity = (uint32_t)std::min<uint64_t>(g->e_part / kPushBigDegree + 1024, 0x7FFFFFFFull);
      LUXB_TRY(gmalloc(g, (PushArgs::BigSeg**)&g->d_big_list, g->big_capacity));
      LUXB_TRY(gmalloc(g, &g->d_fq_all, g->fq_total));
      LUXB_TRY(gmalloc(g, &g->d_fq_new, g->slot_bytes[g->cfg.rank]));
      LUXB_TRY(gmalloc(g, &g->d_fq_tmp, g->slot_bytes[g->cfg.rank]));
      LUXB_TRY(gmalloc(g, &g->d_hdr_all, 2 * LUXB_MAX_PARTS));
      LUXB_TRY(gmalloc(g, &g->h_hdr, 2 * LUXB_MAX_PARTS, MemKind::kPinned));
      LUXB_TRY(gmalloc(g, &g->h_scratch, 16, MemKind::kPinned));
      LUXB_TRY(reset_label_state(g, false, g->cfg.start_vtx));
      if (g->P > 1) {
        // warm the communicator with the collectives the hot loop uses (NCCL sets up channels lazily, ~1 s for the
        // first large grouped broadcast at 8 ranks): re-broadcasting the identical initial labels is a no-op
        LUXB_NCCL(nccl().AllGather(g->d_fq_new, g->d_hdr_all, 8, ncclUint8, g->comm, g->stream));
        LUXB_TRY(allgather_slices(g, g->d_val[0], 4));
        LUXB_CUDA(cudaStreamSynchronize(g->stream));
      }
      if (app_of(g).entry == kBcRun) LUXB_TRY(bc_alloc(g));
      break;
    }
    case LUXB_TC: LUXB_TRY(tc_build(g)); break;
    case LUXB_KCORE: LUXB_TRY(kcore_build(g)); break;
    case LUXB_TRUSS: LUXB_TRY(truss_build(g)); break;
  }
  LUXB_CUDA(cudaStreamSynchronize(g->stream));
  g->cur = 0;
  g->inited = true;
  return 0;
}

// ---- exchange helpers ---------------------------------------------------------------------------------------
// all-gather of unequal slices = one grouped set of in-place broadcasts (root p sends partition p's slice)
static int allgather_slices(luxb_graph* g, void* replica, size_t elem_bytes) {
  if (g->P == 1) return 0;
  LUXB_NCCL(nccl().GroupStart());
  for (int p = 0; p < g->P; ++p) {
    if (g->np[p] == 0) continue;
    char* ptr = reinterpret_cast<char*>(replica) + (size_t)g->rl[p] * elem_bytes;
    LUXB_NCCL(nccl().Broadcast(ptr, ptr, (size_t)g->np[p] * elem_bytes, ncclUint8, p, g->comm, g->stream));
  }
  LUXB_NCCL(nccl().GroupEnd());
  return 0;
}

// iteration barrier of the P2P exchange: a 4-byte all-reduce enqueued after the compute kernels; when it
// completes on a rank, every peer's kernels (and therefore their stores into this rank's replica) are done.
static int p2p_barrier(luxb_graph* g) {
  if (g->P == 1) return 0;
  // the flag kernel is used where it has been validated on hardware (PageRank exchange, 4 GPUs, bit-identical values and the
  // same iteration time as the all-reduce); LUXB_BARRIER=flag extends it to the other apps
  if (g->flag_barrier && g->p2p_ready && (g->cfg.app == LUXB_PAGERANK || g->flag_barrier_all)) {
    FlagBarrierArgs a{};
    for (int p = 0; p < g->P; ++p) a.peer[p] = reinterpret_cast<uint32_t*>(g->peer_flags[p]);
    a.mine = g->d_flags;
    a.err = g->h_barrier_err;
    a.P = g->P;
    a.me = g->cfg.rank;
    a.epoch = ++g->barrier_epoch;
    a.timeout_ns = g->barrier_timeout_ns;
    flag_barrier_kernel<<<1, LUXB_MAX_PARTS, 0, g->stream>>>(a);
    LUXB_CUDA(cudaGetLastError());
    g->stats.kernel_launches++;
    return 0;
  }
  if (!g->d_sync) LUXB_TRY(gmalloc(g, &g->d_sync, 4));
  LUXB_NCCL(nccl().AllReduce(g->d_sync, g->d_sync, 1, ncclUint32, ncclSum, g->comm, g->stream));
  return 0;
}

extern "C++" {
template <class Prog, class Shape>
static int launch_pull_shape(luxb_graph* g, const PullArgs<Prog>& a) {
  auto kern = pull_tile_kernel<Prog, Shape>;
  const int want = g->pull_ctas;
  constexpr size_t smem = pull_smem_bytes<Prog, Shape>();
  // carve out exactly `want` CTAs' worth of shared memory; the rest of the 256 KB unified array stays L1.
  // (function attributes are per device and idempotent: set on every launch, no process-global cache)
  LUXB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  int carve_pct = (int)std::min<size_t>(100, (want * (smem + 1024) * 100 + 228 * 1024 - 1) / (228 * 1024));
  LUXB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributePreferredSharedMemoryCarveout, carve_pct));
  const uint32_t n_super = (a.n_tiles + Shape::kWarps - 1) / Shape::kWarps;
  uint32_t grid = (uint32_t)std::min<uint64_t>((uint64_t)g->num_sms * want, n_super);
  kern<<<grid, Shape::kThreads, smem, g->stream>>>(a);
  LUXB_CUDA(cudaGetLastError());
  return 0;
}

static int kt_begin(luxb_graph* g) {
  if (!g->kernel_timing) return 0;
  if (g->kt_used + 2 > g->kt_events.size()) {
    cudaEvent_t e0, e1;
    LUXB_CUDA(cudaEventCreate(&e0));
    LUXB_CUDA(cudaEventCreate(&e1));
    g->kt_events.push_back(e0);
    g->kt_events.push_back(e1);
  }
  LUXB_CUDA(cudaEventRecord(g->kt_events[g->kt_used], g->stream));
  return 0;
}
static int kt_end(luxb_graph* g) {
  if (!g->kernel_timing) return 0;
  LUXB_CUDA(cudaEventRecord(g->kt_events[g->kt_used + 1], g->stream));
  g->kt_used += 2;
  return 0;
}

template <class Prog>
static void fill_fixup_args(PullArgs<Prog>& a, const FixupScratch& f) {
  a.head_partial = reinterpret_cast<typename Prog::Acc*>(f.d_head);
  a.tail_partial = reinterpret_cast<typename Prog::Acc*>(f.d_tail);
  a.carry = reinterpret_cast<typename Prog::Wide*>(f.d_carry);
  a.carry_flag = f.d_carry_flag;
  a.block_agg = reinterpret_cast<typename Prog::Wide*>(f.d_block_agg);
  a.block_flag = f.d_block_flag;
}

// f is the sweep's own scratch (the fused fix-up keeps its launch epoch there); st: the stream of the swept kernel
template <class Prog>
static int launch_fixup(luxb_graph* g, const PullArgs<Prog>& a, FixupScratch& f, const uint2* piece_slot = nullptr,
                        cudaStream_t st = nullptr) {
  if (a.n_tiles <= 1) return 0;
  if (!st) st = g->stream;
  if (g->fused_fixup) {
    if (!f.d_chain) {
      LUXB_TRY(gmalloc(g, &f.d_chain, 4ull * f.n_fix_blocks + 4));  // values, status words, [4 n] = ticket counter
      LUXB_CUDA(cudaMemsetAsync(f.d_chain, 0, (4ull * f.n_fix_blocks + 4) * 8, st));
      f.chain_epoch = 0;
    }
    FixupChain<Prog> ch;
    ch.value = f.d_chain;
    ch.status = f.d_chain + 2ull * f.n_fix_blocks;
    ch.ticket = f.d_chain + 4ull * f.n_fix_blocks;
    ch.n_blocks = f.n_fix_blocks;
    ch.epoch = ++f.chain_epoch;
    if (f.chain_epoch >= 0x3FFFFFF0u) {  // 30-bit epochs: start over with a clean status array
      LUXB_CUDA(cudaMemsetAsync(f.d_chain, 0, (4ull * f.n_fix_blocks + 4) * 8, st));
      f.chain_epoch = ch.epoch = 1;
    }
    pull_fixup_fused_kernel<Prog><<<f.n_fix_blocks, kFixBlock, 0, st>>>(a, ch, piece_slot);
    LUXB_CUDA(cudaGetLastError());
    g->stats.kernel_launches++;
    return 0;
  }
  pull_fixup_scan_kernel<Prog><<<f.n_fix_blocks, kFixBlock, 0, st>>>(a);
  pull_fixup_blocks_kernel<Prog><<<1, 1024, 0, st>>>(a, f.n_fix_blocks);
  pull_fixup_apply_kernel<Prog><<<f.n_fix_blocks, kFixBlock, 0, st>>>(a, piece_slot);
  LUXB_CUDA(cudaGetLastError());
  g->stats.kernel_launches += 3;
  return 0;
}

// one pull sweep over layout L gathering through the ids `src`.  hub_bits != nullptr: those vertices get their raw sum
// (panel.cuh).
template <class Prog>
static int launch_pull(luxb_graph* g, PullLayout& L, const uint32_t* src, const typename Prog::Vertex* x_nat,
                       const typename Prog::Vertex* x_cold, const typename Prog::Vertex* x_hot, uint32_t hot_n,
                       typename Prog::Vertex* out_local, const typename Prog::Params& prm, const uint32_t* hub_bits = nullptr,
                       bool timed = true) {
  if (L.n_tiles == 0) return 0;
  PullArgs<Prog> a{};
  a.row_end = L.d_row_end;
  a.row_end32 = L.d_row_end32;
  a.src = src;
  a.x_nat = x_nat;
  a.n_part = L.n_vtx;
  a.e_part = L.e_cnt;
  a.row_left = g->row_left;
  a.x_old = x_cold;  // gather ids >= hot_n index this array at (id - hot_n)
  a.x_hot = x_hot;
  a.hot_n = hot_n;
  a.out = out_local;
  a.tile_v = L.d_tile_v;
  a.n_tiles = L.n_tiles;
  fill_fixup_args(a, L.fix);
  a.tile_counter = reinterpret_cast<uint32_t*>(g->d_counters + 2);
  LUXB_CUDA(cudaMemsetAsync(a.tile_counter, 0, 4, g->stream));
  a.prm = prm;
  a.hub_bits = hub_bits;
  a.raw_out = 0;
  if constexpr (Prog::kWeighted) a.weight = g->d_weight;  // CSC order = the order of src (base layout only)
  if (timed) LUXB_TRY(kt_begin(g));
  switch (g->pull_shape) {
#define LUXB_CASE_SHAPE(id, ipt, warps, stages) \
    case id: LUXB_TRY((launch_pull_shape<Prog, PullShape##id>(g, a))); break;
    LUXB_PULL_SHAPES(LUXB_CASE_SHAPE)
    default: set_error("bad pull shape"); return LUXB_ERR_STATE;
  }
  if (timed) LUXB_TRY(kt_end(g));
  g->stats.kernel_launches++;
  pt_mark(g, 0);
  LUXB_TRY(launch_fixup(g, a, L.fix));
  pt_mark(g, 1);
  return 0;
}
}  // extern "C++"

// ---- flagged segmented-scan sweep (seg.cuh) and its source-blocked variant (panel.cuh) ------------------------------
// shapes <consumer warps, ring stages, rounds of 256 edges per warp piece>
#define LUXB_SEG_MAIN_SHAPES(X) X(0, 8, 2, 2) X(1, 8, 3, 1) X(2, 12, 2, 1) X(3, 8, 2, 4) X(4, 16, 2, 1) X(5, 8, 4, 1) X(6, 8, 2, 1) X(7, 6, 2, 2)
#define LUXB_DECL_MSHAPE(id, warps, stages, rounds) using SegMain##id = SegShape<warps, stages, rounds, false, 0>;
LUXB_SEG_MAIN_SHAPES(LUXB_DECL_MSHAPE)
// panel shapes: + shared-memory table capacity (values, <= 32768: 15-bit offsets); one CTA per SM
// (..., edges per lane and round)
#define LUXB_SEG_PANEL_SHAPES(X) \
  X(0, 31, 2, 2, 32768, 8) X(1, 24, 2, 1, 32768, 16) X(2, 16, 2, 2, 32768, 16) X(3, 24, 2, 2, 32768, 8) X(4, 20, 2, 1, 32768, 16) X(5, 16, 2, 4, 32768, 8)
#define LUXB_DECL_PSHAPE(id, warps, stages, rounds, tab, v) using SegPanel##id = SegShape<warps, stages, rounds, true, tab, v>;
LUXB_SEG_PANEL_SHAPES(LUXB_DECL_PSHAPE)
struct SegShapeInfo { int piece, stage_edges, tab; };
#define LUXB_MSHAPE_INFO(id, warps, stages, rounds) {SegMain##id::kPiece, SegMain##id::kStageEdges, 0},
#define LUXB_PSHAPE_INFO(id, warps, stages, rounds, tab, v) {SegPanel##id::kPiece, SegPanel##id::kStageEdges, SegPanel##id::kTab},
static const SegShapeInfo kSegMainInfo[] = {LUXB_SEG_MAIN_SHAPES(LUXB_MSHAPE_INFO)};
static const SegShapeInfo kSegPanelInfo[] = {LUXB_SEG_PANEL_SHAPES(LUXB_PSHAPE_INFO)};
static const int kNumSegMain = sizeof(kSegMainInfo) / sizeof(SegShapeInfo);
static const int kNumSegPanel = sizeof(kSegPanelInfo) / sizeof(SegShapeInfo);

static int env_int(const char* name, int dflt) {
  const char* e = getenv(name);
  return e ? atoi(e) : dflt;
}

static double env_double(const char* name, double dflt) {
  const char* e = getenv(name);
  return e ? atof(e) : dflt;
}

// the only reader of these variables; a shape out of range falls back to shape 0
static void resolve_sweep_settings(SweepSettings& s) {
  s = SweepSettings();
  if (const char* e = getenv("LUXB_SWEEP")) s.seg = strcmp(e, "merge") != 0;
  auto shape = [](const char* name, int dflt, int n) { const int v = env_int(name, dflt); return v < 0 || v >= n ? 0 : v; };
  s.main_shape = shape("LUXB_SEG_MAIN_SHAPE", s.main_shape, kNumSegMain);
  s.panel_shape = shape("LUXB_SEG_PANEL_SHAPE", s.panel_shape, kNumSegPanel);
  s.cs_shape = shape("LUXB_CS_SHAPE", s.main_shape, kNumSegMain);
  s.sb = env_int("LUXB_SB", s.sb);
  const int tab = kSegPanelInfo[s.panel_shape].tab;
  s.sb_bs = std::min<uint32_t>((uint32_t)std::max(4, env_int("LUXB_SB_BS", tab)) & ~3u, (uint32_t)tab);
  s.sb_blocks = (uint32_t)std::min(std::max(env_int("LUXB_SB_BLOCKS", (int)s.sb_blocks), 1), kPanelMaxBlocks);
  s.sb_min_indeg = (uint32_t)std::max(env_int("LUXB_SB_MIN_INDEG", (int)s.sb_min_indeg), 1);
  s.sb_tier = env_int("LUXB_SB_TIER", s.sb_tier);
  s.sb_slot_edges = env_double("LUXB_SB_SLOT_EDGES", s.sb_slot_edges);
  s.cs = env_int("LUXB_CS", s.cs);
  s.cs_seg_mb = env_double("LUXB_CS_SEG_MB", s.cs_seg_mb);
  s.hot_mb = env_double("LUXB_HOT_MB", s.hot_mb);
  s.l2_persist = env_int("LUXB_L2_PERSIST", 1) != 0;
  s.l2_window_mb = env_double("LUXB_L2_WINDOW_MB", s.l2_window_mb);
  s.panel_sms = std::max(0, env_int("LUXB_PANEL_SMS", s.panel_sms));
}

extern "C++" {
// Build the flagged stream of a CSC (seg.cuh).  row_end: inclusive end offsets (u64) of n_vtx "vertices" whose edges,
// in CSC order, carry the gather ids `ids`; blk: the vertex / edge ranges of the blocks (one block = plain stream;
// wbase / hshift are filled here).  Every block is padded with 1 .. stage_edges head-flagged dummy words to a whole
// number of stages.  On return L holds words, close list, tile_v (heads before each piece), fix-up scratch and, if
// want_empty, the list of vertices without edges.  super_end (optional) receives the first stage after each block.
// slots: a group stream (panel.cuh) — no close list; its non-empty "vertices" are the compact slots slot_base,
// slot_base + 1, ... in order, L.d_piece_slot says which of them each piece closes and L.n_slots counts them.
template <class Word, class In>
static int build_seg_stream(luxb_graph* g, PullLayout& L, const uint64_t* d_row_end, uint32_t n_vtx, const In* d_ids, uint64_t e_cnt,
                            StreamBlocks& blk, uint32_t stage_edges, uint32_t piece, bool want_empty, const uint32_t* hub_bits,
                            uint32_t* super_end, bool slots = false, uint32_t slot_base = 0) {
  const int grid = g->num_sms * 8;
  DevTmp tmp;
  L = PullLayout();
  L.n_vtx = n_vtx;
  L.e_cnt = e_cnt;
  uint64_t words = 0, pads_total = 0;
  for (uint32_t b = 0; b < blk.n_blocks; ++b) {
    const uint64_t eb = blk.ebase[b + 1] - blk.ebase[b];
    const uint64_t pad = stage_edges - eb % stage_edges;  // 1 .. stage_edges: the first pad closes the block's last vertex
    blk.wbase[b] = words;
    blk.hshift[b] = pads_total;
    words += eb + pad;
    pads_total += pad;
    if (super_end) super_end[b] = (uint32_t)(words / stage_edges);
  }
  blk.wbase[blk.n_blocks] = words;
  blk.hshift[blk.n_blocks] = pads_total;
  LUXB_ARG(words / piece < 0xFFFFFFF0ull && words / stage_edges < 0xFFFFFFF0ull, "stream too large");
  L.n_words = words;
  L.n_stages = (uint32_t)(words / stage_edges);
  L.n_tiles = (uint32_t)(words / piece);
  // 1. non-empty vertices and their rank
  uint32_t *d_flag = nullptr, *d_rank = nullptr;
  LUXB_TRY(tmp.alloc(&d_flag, (uint64_t)n_vtx + 1));
  LUXB_TRY(tmp.alloc(&d_rank, (uint64_t)n_vtx + 1));
  nonempty_flag_kernel<<<grid, 256, 0, g->stream>>>(d_row_end, n_vtx, d_flag);
  LUXB_CUDA(cudaMemsetAsync(d_flag + n_vtx, 0, 4, g->stream));
  LUXB_TRY(cub_call(tmp, g->stream, [&](void* t, size_t& b) {
    return cub::DeviceScan::ExclusiveSum(t, b, d_flag, d_rank, (int)n_vtx + 1, g->stream);
  }));
  uint32_t n_seg = 0;
  LUXB_CUDA(cudaMemcpyAsync(&n_seg, d_rank + n_vtx, 4, cudaMemcpyDeviceToHost, g->stream));
  LUXB_CUDA(cudaStreamSynchronize(g->stream));
  // 2. words: ids, then pads, then head flags; close list (entry j + 1 = owner of head j, dummies for the pads) unless
  // the heads close compact slots
  Word* d_words = nullptr;
  LUXB_TRY(gmalloc(g, &d_words, words + 64));
  L.d_src = d_words;
  if (e_cnt) stream_copy_kernel<Word, In><<<grid, 256, 0, g->stream>>>(d_ids, e_cnt, blk, d_words);
  for (uint32_t b = 0; b < blk.n_blocks; ++b) {
    const uint64_t from = blk.wbase[b] + (blk.ebase[b + 1] - blk.ebase[b]);
    stream_pad_kernel<Word><<<grid_for(blk.wbase[b + 1] - from, 256, grid), 256, 0, g->stream>>>(d_words, from, blk.wbase[b + 1]);
  }
  LUXB_CUDA(cudaGetLastError());
  const uint64_t n_heads = (uint64_t)n_seg + pads_total;
  LUXB_ARG(n_heads < 0xFFFFFFF0ull, "too many segments");
  if (!slots) {
    LUXB_TRY(gmalloc(g, &L.d_close, n_heads + 2));
    LUXB_CUDA(cudaMemsetAsync(L.d_close, 0xFF, (n_heads + 2) * 4, g->stream));
  }
  stream_heads_kernel<Word><<<grid, 256, 0, g->stream>>>(d_row_end, n_vtx, d_flag, d_rank, blk, d_words, L.d_close);
  LUXB_CUDA(cudaGetLastError());
  // 3. heads before each piece
  uint32_t* d_cnt = nullptr;
  LUXB_TRY(tmp.alloc(&d_cnt, (uint64_t)L.n_tiles + 2));
  LUXB_CUDA(cudaMemsetAsync(d_cnt, 0, ((size_t)L.n_tiles + 2) * 4, g->stream));
  piece_heads_kernel<Word><<<grid, 256, 0, g->stream>>>(d_words, L.n_tiles, piece, d_cnt);
  LUXB_CUDA(cudaGetLastError());
  LUXB_TRY(gmalloc(g, &L.d_tile_v, (uint64_t)L.n_tiles + 2));
  LUXB_TRY(cub_call(tmp, g->stream, [&](void* t, size_t& b) {
    return cub::DeviceScan::ExclusiveSum(t, b, d_cnt, L.d_tile_v, (int)L.n_tiles + 1, g->stream);
  }));
  uint32_t heads_counted = 0;
  LUXB_CUDA(cudaMemcpyAsync(&heads_counted, L.d_tile_v + L.n_tiles, 4, cudaMemcpyDeviceToHost, g->stream));
  if (slots) {
    LUXB_ARG((uint64_t)slot_base + n_seg < 0x7FFFFFF0ull, "too many slots");
    LUXB_TRY(gmalloc(g, &L.d_piece_slot, (uint64_t)L.n_tiles + 1));
    piece_slot_kernel<<<grid_for(L.n_tiles, 256, grid), 256, 0, g->stream>>>(L.d_tile_v, L.n_tiles, piece, d_rank, blk, slot_base, L.d_piece_slot);
    LUXB_CUDA(cudaGetLastError());
    L.n_slots = n_seg;
  }
  // 4. vertices without edges (hubs among them apart)
  unsigned int* d_cur2 = nullptr;
  if (want_empty) {
    const uint32_t n_e = n_vtx - n_seg;
    LUXB_TRY(gmalloc(g, &L.d_empty, (uint64_t)n_e + 1));
    LUXB_TRY(gmalloc(g, &L.d_empty_hub, (uint64_t)n_e + 1));
    LUXB_TRY(tmp.alloc(&d_cur2, 2));
    LUXB_CUDA(cudaMemsetAsync(d_cur2, 0, 8, g->stream));
    empty_split_kernel<<<grid, 256, 0, g->stream>>>(d_flag, n_vtx, hub_bits, L.d_empty, L.d_empty_hub, d_cur2);
    LUXB_CUDA(cudaGetLastError());
    unsigned int h_cur2[2] = {0, 0};
    LUXB_CUDA(cudaMemcpyAsync(h_cur2, d_cur2, 8, cudaMemcpyDeviceToHost, g->stream));
    LUXB_CUDA(cudaStreamSynchronize(g->stream));
    L.n_empty = h_cur2[0];
    L.n_empty_hub = h_cur2[1];
  }
  LUXB_CUDA(cudaStreamSynchronize(g->stream));
  if ((uint64_t)heads_counted != n_heads) {
    set_error("flagged stream: %u heads counted, %llu expected", heads_counted, (unsigned long long)n_heads);
    return LUXB_ERR_STATE;
  }
  // 5. fix-up scratch
  return alloc_fixup(g, L.fix, L.n_tiles);
}
}  // extern "C++"

// the main stream sb_main: every local vertex over the CSC (row_end, ids) of the edges left to it (all of them without
// the source-blocked split; hub_bits then null)
static int build_main_stream(luxb_graph* g, const uint64_t* d_row_end, const uint32_t* d_ids, uint64_t e_cnt, const uint32_t* hub_bits) {
  const SegShapeInfo shp = kSegMainInfo[g->sweep.main_shape];
  StreamBlocks blk{};
  blk.n_blocks = 1;
  blk.vfirst[1] = g->n_part;
  blk.ebase[1] = e_cnt;
  return build_seg_stream<uint32_t, uint32_t>(g, g->sb_main, d_row_end, g->n_part, d_ids, e_cnt, blk, (uint32_t)shp.stage_edges,
                                              (uint32_t)shp.piece, true, hub_bits, nullptr);
}

extern "C++" {
// The flagged stream of the split's groups [g0, g1) (panel.cuh): their e_cnt sorted edges (d_key / d_pay) -> ids
// (group_fill_kernel), the CSC over their dense (group, hub) pairs vbase[g0] .. vbase[g1] - 1, their words of the slot
// bitmap d_bits, and the stream, whose heads close the compact slots slot_base, slot_base + 1, ... (the non-empty pairs
// in order).  With super_end every group is padded to whole stages (the panel: a stage never straddles two source
// blocks) and super_end receives the first stage after each; without, the groups form one block.
template <class Word>
static int build_group_stream(luxb_graph* g, PullLayout& L, const uint16_t* d_key, const uint64_t* d_pay, uint64_t e_cnt, uint32_t g0,
                              uint32_t g1, const unsigned long long* hist, uint32_t bs, const SegShapeInfo& shp, uint32_t* super_end,
                              uint32_t* d_bits, uint32_t slot_base) {
  const int grid = g->num_sms * 8;
  const uint32_t* vbase = g->sb_groups.vbase;
  const uint32_t v0 = vbase[g0], n_vtx = vbase[g1] - v0;
  DevTmp tmp;
  Word* d_ids = nullptr;
  uint32_t* d_vcount = nullptr;
  uint64_t* d_vrow = nullptr;
  LUXB_TRY(tmp.alloc(&d_ids, e_cnt + 32));
  LUXB_TRY(tmp.alloc(&d_vcount, (uint64_t)n_vtx + 1));
  LUXB_CUDA(cudaMemsetAsync(d_vcount, 0, ((size_t)n_vtx + 1) * 4, g->stream));
  group_fill_kernel<Word><<<grid, 256, 0, g->stream>>>(d_key, d_pay, e_cnt, g->d_src_gather, bs, g->sb_groups, v0, d_ids, d_vcount);
  LUXB_CUDA(cudaGetLastError());
  LUXB_TRY(tmp.alloc(&d_vrow, (uint64_t)n_vtx + 4));
  widen_u32_to_u64_kernel<<<grid, 256, 0, g->stream>>>(d_vcount, d_vrow, n_vtx);
  LUXB_TRY(cub_call(tmp, g->stream, [&](void* t, size_t& b) {
    return cub::DeviceScan::InclusiveSum(t, b, d_vrow, d_vrow, (int)n_vtx, g->stream);
  }));
  slot_bits_kernel<<<grid, 256, 0, g->stream>>>(d_vcount, g->sb_groups, g0, g1, v0, d_bits);
  LUXB_CUDA(cudaGetLastError());
  tmp.release(d_vcount);
  StreamBlocks blk{};
  blk.n_blocks = super_end ? g1 - g0 : 1;
  for (uint32_t b = 0; b < blk.n_blocks; ++b) {
    blk.vfirst[b + 1] = super_end ? vbase[g0 + b + 1] - v0 : n_vtx;
    blk.ebase[b + 1] = super_end ? blk.ebase[b] + hist[g0 + b] : e_cnt;
  }
  return build_seg_stream<Word, Word>(g, L, d_vrow, n_vtx, d_ids, e_cnt, blk, (uint32_t)shp.stage_edges, (uint32_t)shp.piece, false,
                                      nullptr, super_end, true, slot_base);
}
}  // extern "C++"

// Split this partition's (hot-packed) CSC into the panel (hot source block x hub destination, 15-bit offsets, gathered
// from shared memory), with the compact cold values of one rank (cold_z) the cold-hub stream (cold source segment x hub
// destination, panel.cuh, ColdSplit), and the main stream (everything else, gathered through L1).  Settings and their
// automatic rules: SweepSettings.
static int build_panel_layout(luxb_graph* g) {
  g->sb_on = false;
  g->cs_on = false;
  const SweepSettings& st = g->sweep;
  if (!split_may_run(g) || g->hot_n == 0 || g->e_part == 0 || g->e_part >= 0xFFFFFFFFull) return 0;
  const SegShapeInfo shp = kSegPanelInfo[st.panel_shape];
  const uint32_t bs = st.sb_bs;
  const uint32_t NB0 = (uint32_t)((std::min<uint64_t>(g->hot_n, (uint64_t)st.sb_blocks * bs) + bs - 1) / bs);  // tier 0
  const bool tiers = st.sb_tier > 0 || (st.sb_tier < 0 && g->cold_z && g->e_part >= kSplitMinEdges);
  const uint32_t nb_all = tiers ? (uint32_t)std::min<uint64_t>(((uint64_t)g->hot_n + bs - 1) / bs, kPanelMaxBlocks) : NB0;
  const int grid = g->num_sms * 8;
  DevTmp tmp;

  // 1. hub destinations
  uint32_t *d_flag = nullptr, *d_hub_idx = nullptr;
  LUXB_TRY(tmp.alloc(&d_flag, (uint64_t)g->n_part + 1));
  LUXB_TRY(tmp.alloc(&d_hub_idx, (uint64_t)g->n_part + 1));
  hub_flag_kernel<<<grid, 256, 0, g->stream>>>(g->d_row_end, g->n_part, st.sb_min_indeg, d_flag);
  LUXB_CUDA(cudaGetLastError());
  LUXB_TRY(cub_call(tmp, g->stream, [&](void* t, size_t& b) {
    return cub::DeviceScan::ExclusiveSum(t, b, d_flag, d_hub_idx, (int)g->n_part, g->stream);
  }));
  uint32_t last_idx = 0, last_flag = 0;
  LUXB_CUDA(cudaMemcpyAsync(&last_idx, d_hub_idx + g->n_part - 1, 4, cudaMemcpyDeviceToHost, g->stream));
  LUXB_CUDA(cudaMemcpyAsync(&last_flag, d_flag + g->n_part - 1, 4, cudaMemcpyDeviceToHost, g->stream));
  LUXB_CUDA(cudaStreamSynchronize(g->stream));
  const uint32_t Nh = last_idx + last_flag;
  if (Nh == 0 || (uint64_t)Nh * NB0 >= 0x7FFFFFF0ull) return 0;
  uint32_t *d_hub_vtx = nullptr, *d_hub_bits = nullptr, *d_cov = nullptr;
  LUXB_TRY(tmp.alloc(&d_hub_vtx, Nh));
  LUXB_TRY(tmp.alloc(&d_hub_bits, ((uint64_t)g->n_part + 31) / 32 + 1));
  LUXB_TRY(tmp.alloc(&d_cov, Nh));
  hub_list_kernel<<<grid, 256, 0, g->stream>>>(d_flag, d_hub_idx, g->n_part, d_hub_vtx, d_hub_bits);
  LUXB_CUDA(cudaGetLastError());
  // hubs by in-degree, descending: the hub prefix of every block holds the hubs of highest in-degree
  std::vector<uint32_t> hub_key(Nh);  // ~in-degree, ascending
  {
    uint32_t *d_hkey = nullptr, *d_hkey2 = nullptr, *d_hvtx2 = nullptr;
    LUXB_TRY(tmp.alloc(&d_hkey, Nh));
    LUXB_TRY(tmp.alloc(&d_hkey2, Nh));
    LUXB_TRY(tmp.alloc(&d_hvtx2, Nh));
    hub_order_key_kernel<<<grid, 256, 0, g->stream>>>(g->d_row_end, d_hub_vtx, Nh, d_hkey);
    LUXB_CUDA(cudaGetLastError());
    LUXB_TRY(cub_call(tmp, g->stream, [&](void* t, size_t& b) {
      return cub::DeviceRadixSort::SortPairs(t, b, d_hkey, d_hkey2, d_hub_vtx, d_hvtx2, (int)Nh, 0, 32, g->stream);
    }));
    LUXB_CUDA(cudaMemcpyAsync(d_hub_vtx, d_hvtx2, (size_t)Nh * 4, cudaMemcpyDeviceToDevice, g->stream));
    hub_pos_kernel<<<grid, 256, 0, g->stream>>>(d_hub_vtx, Nh, d_hub_idx);
    LUXB_CUDA(cudaGetLastError());
    LUXB_CUDA(cudaMemcpyAsync(hub_key.data(), d_hkey2, (size_t)Nh * 4, cudaMemcpyDeviceToHost, g->stream));
    LUXB_CUDA(cudaStreamSynchronize(g->stream));
    tmp.release(d_hkey);
    tmp.release(d_hkey2);
    tmp.release(d_hvtx2);
  }
  // hub prefix N_b of every block: all hubs in the first keying
  uint32_t NB = nb_all;
  std::vector<uint32_t> n_pref(NB, Nh);
  uint32_t* d_pref = nullptr;
  LUXB_TRY(tmp.alloc(&d_pref, kPanelMaxBlocks));
  LUXB_CUDA(cudaMemcpyAsync(d_pref, n_pref.data(), (size_t)NB * 4, cudaMemcpyHostToDevice, g->stream));

  // cold segments: cold gather ids [H, H + C) cut into S <= 255 - NB0 segments of `seg` values, groups NB .. NB + S - 1
  ColdSplit cs{};
  cs.hot_n = g->hot_n;
  cs.key0 = NB;
  uint32_t S = 0;
  if (g->cold_z && st.cs != 0 && g->cold_n > 0) {
    const uint32_t s_max = 255 - NB0;
    uint64_t seg = std::max<uint64_t>(1, (uint64_t)(st.cs_seg_mb * 1e6 / 4.0));
    seg = std::min<uint64_t>(std::max<uint64_t>(seg, (g->cold_n + s_max - 1) / s_max), g->cold_n);
    const uint32_t n_seg = (uint32_t)((g->cold_n + seg - 1) / seg);
    if ((uint64_t)Nh * n_seg < 0x7FFFFFF0ull) { cs.seg = (uint32_t)seg; S = n_seg; }
  }

  // 2. edge keys: the group of the edge for (hot source, hub destination in the block's prefix) and (cold source, hub
  // destination) edges, kSplitKeyMain for the rest; then the key histogram
  uint16_t *d_key = nullptr, *d_key2 = nullptr;
  uint64_t *d_pay = nullptr, *d_pay2 = nullptr;
  LUXB_TRY(tmp.alloc(&d_key, g->e_part));
  LUXB_TRY(tmp.alloc(&d_key2, g->e_part));
  LUXB_TRY(tmp.alloc(&d_pay, g->e_part));
  LUXB_TRY(tmp.alloc(&d_pay2, g->e_part));
  constexpr int kBins = kSplitKeyMain + 1;
  unsigned long long* d_hist = nullptr;
  LUXB_TRY(tmp.alloc(&d_hist, kBins));
  unsigned long long hist[kBins];
  auto key_edges = [&]() -> int {
    const uint32_t n_src = (uint32_t)std::min<uint64_t>(g->hot_n, (uint64_t)NB * bs);
    edge_iota_kernel<<<grid, 256, 0, g->stream>>>(d_pay, d_key, g->e_part);
    hub_key_kernel<<<grid, 256, 0, g->stream>>>(g->d_row_end, g->d_src_gather, d_hub_vtx, Nh, n_src, bs, d_pref, NB, d_key, d_pay, d_cov, cs);
    LUXB_CUDA(cudaMemsetAsync(d_hist, 0, kBins * 8, g->stream));
    key_hist_kernel<<<grid, 256, 0, g->stream>>>(d_key, g->e_part, d_hist);
    LUXB_CUDA(cudaGetLastError());
    LUXB_CUDA(cudaMemcpyAsync(hist, d_hist, sizeof(hist), cudaMemcpyDeviceToHost, g->stream));
    LUXB_CUDA(cudaStreamSynchronize(g->stream));
    return 0;
  };
  LUXB_TRY(key_edges());
  // Both decisions come from this first histogram.  Tiers: block b >= NB0 keeps hub h while d_h * m_b >= slot_edges,
  // m_b = (edges block b -> hubs) / (edges into hubs).  Cold-hub verdict: a cold key only needs a cold source (never
  // below n_src) and a hub destination, so fewer blocks renumber the segments without moving an edge.
  bool rekey = false;
  if (tiers && NB > NB0) {
    uint64_t e_hub = 0;
    for (uint32_t h = 0; h < Nh; ++h) e_hub += ~hub_key[h];
    for (uint32_t b = NB0; b < NB; ++b) {
      uint32_t keep = 0;
      if (hist[b] > 0) {
        const double d_min = st.sb_slot_edges * (double)e_hub / (double)hist[b];
        // hub_key ascends (~in-degree): the hubs with in-degree >= d_min are a prefix
        keep = (uint32_t)(std::partition_point(hub_key.begin(), hub_key.end(), [&](uint32_t k) { return (double)~k >= d_min; }) - hub_key.begin());
      }
      n_pref[b] = std::min(keep, n_pref[b - 1]);
      rekey |= n_pref[b] < Nh;
    }
    while (NB > NB0 && n_pref[NB - 1] == 0) --NB;
    cs.key0 = NB;
    LUXB_CUDA(cudaMemcpyAsync(d_pref, n_pref.data(), (size_t)NB * 4, cudaMemcpyHostToDevice, g->stream));
  }
  uint64_t e_cs = 0;
  for (uint32_t s = 0; s < S; ++s) e_cs += hist[nb_all + s];
  if (S && st.cs < 0 && !(e_cs > 0 && (double)e_cs >= kColdSplitMinShare * (double)g->e_part)) {
    rekey |= e_cs > 0;  // automatic and too few cold -> hub edges: no cold split
    cs.seg = 0;
    S = 0;
  }
  if (rekey) LUXB_TRY(key_edges());
  {
    // 3. two stable sorts: by hub position (payload bits 32.., 0 for main edges), then by key.  Every group then lists
    // its edges by slot (hub order is not id order), the main stream keeps the CSC order.
    cub::DoubleBuffer<uint16_t> kb(d_key, d_key2);
    cub::DoubleBuffer<uint64_t> pb(d_pay, d_pay2);
    int hbits = 1;
    while ((1ull << hbits) < (uint64_t)Nh) ++hbits;
    LUXB_TRY(cub_call(tmp, g->stream, [&](void* t, size_t& b) {
      return cub::DeviceRadixSort::SortPairs(t, b, pb, kb, (long long)g->e_part, 32, 32 + hbits, g->stream);
    }));
    LUXB_TRY(cub_call(tmp, g->stream, [&](void* t, size_t& b) {
      return cub::DeviceRadixSort::SortPairs(t, b, kb, pb, (long long)g->e_part, 0, kSplitKeyBits, g->stream);
    }));
    tmp.release(kb.Alternate());
    tmp.release(pb.Alternate());
    d_key2 = kb.Current();
    d_pay2 = pb.Current();
  }
  uint64_t e_cov = 0, e_cov0 = 0, e_cold = 0;
  for (uint32_t b = 0; b < NB; ++b) e_cov += hist[b];
  for (uint32_t b = 0; b < NB0; ++b) e_cov0 += hist[b];
  for (uint32_t s = 0; s < S; ++s) e_cold += hist[NB + s];
  const uint64_t e_main = hist[kSplitKeyMain];
  if (e_cov + e_cold + e_main != g->e_part) {
    set_error("panel split lost edges (%llu + %llu + %llu != %llu)", (unsigned long long)e_cov, (unsigned long long)e_cold,
              (unsigned long long)e_main, (unsigned long long)g->e_part);
    return LUXB_ERR_STATE;
  }
  if (e_cov == 0 || (st.sb < 0 && e_cov < g->e_part / 5)) return 0;

  // 4. the group table: block b serves N_b hubs, a cold segment all Nh; dense pair vbase[g] + h, bitmap words from
  // wbase[g]
  const uint32_t NG = NB + S;
  LUXB_ARG(NG < kSplitKeyMain, "panel: too many source groups");
  uint64_t n_pairs = 0, n_words = 0;
  g->sb_groups = SplitGroups{};
  for (uint32_t k = 0; k < NG; ++k) {
    const uint32_t n_k = k < NB ? n_pref[k] : Nh;
    n_pairs += n_k;
    n_words += (n_k + 31) / 32;
    LUXB_ARG(n_pairs < 0x7FFFFFF0ull, "panel: too many (group, hub) pairs");
    g->sb_groups.vbase[k + 1] = (uint32_t)n_pairs;
    g->sb_groups.wbase[k + 1] = (uint32_t)n_words;
  }
  uint32_t *d_slot_bits = nullptr, *d_slot_pre = nullptr;
  LUXB_TRY(tmp.alloc(&d_slot_bits, n_words + 1));
  LUXB_TRY(tmp.alloc(&d_slot_pre, n_words + 1));
  // 5. the panel (per-block stage padding) and the cold-hub stream (one block: its kernel claims stages in order, so the
  // SMs move through the segments together); the cold-hub slots follow the panel's
  LUXB_TRY(build_group_stream<uint16_t>(g, g->sb_panel, d_key2, d_pay2, e_cov, 0, NB, hist, bs, shp, g->sb_super_end, d_slot_bits, 0));
  if (S)
    LUXB_TRY(build_group_stream<uint32_t>(g, g->sb_cold, d_key2 + e_cov, d_pay2 + e_cov, e_cold, NB, NG, hist, 0,
                                          kSegMainInfo[st.cs_shape], nullptr, d_slot_bits, g->sb_panel.n_slots));
  const uint64_t n_slots = (uint64_t)g->sb_panel.n_slots + (S ? g->sb_cold.n_slots : 0);
  // the combine's prefix: slots before each bitmap word, = the streams' numbering
  popc_kernel<<<grid, 256, 0, g->stream>>>(d_slot_bits, n_words, d_slot_pre);
  LUXB_CUDA(cudaMemsetAsync(d_slot_pre + n_words, 0, 4, g->stream));
  LUXB_CUDA(cudaGetLastError());
  LUXB_TRY(cub_call(tmp, g->stream, [&](void* t, size_t& b) {
    return cub::DeviceScan::ExclusiveSum(t, b, d_slot_pre, d_slot_pre, (int)n_words + 1, g->stream);
  }));
  uint32_t kind_slots[4] = {0, 0, 0, 0};  // slots before tier 0, the tiers, the cold segments, the end
  const uint32_t kind_word[4] = {0, g->sb_groups.wbase[NB0], g->sb_groups.wbase[NB], (uint32_t)n_words};
  for (int i = 0; i < 4; ++i) LUXB_CUDA(cudaMemcpyAsync(&kind_slots[i], d_slot_pre + kind_word[i], 4, cudaMemcpyDeviceToHost, g->stream));
  LUXB_CUDA(cudaStreamSynchronize(g->stream));
  if ((uint64_t)kind_slots[3] != n_slots) {
    set_error("panel split: %u slots in the bitmap, %llu in the streams", kind_slots[3], (unsigned long long)n_slots);
    return LUXB_ERR_STATE;
  }

  // 6. main stream: what is left, in the original (dst, src) order
  uint32_t* d_main_src = nullptr;
  uint64_t* d_main_row = nullptr;
  LUXB_TRY(tmp.alloc(&d_main_src, e_main + 8));
  main_fill_kernel<<<grid, 256, 0, g->stream>>>(d_pay2 + e_cov + e_cold, e_main, g->d_src_gather, d_main_src);
  LUXB_TRY(tmp.alloc(&d_main_row, (uint64_t)g->n_part + 4));
  main_indeg_kernel<<<grid, 256, 0, g->stream>>>(g->d_row_end, g->n_part, d_flag, d_hub_idx, d_cov, d_main_row);
  LUXB_CUDA(cudaGetLastError());
  LUXB_TRY(cub_call(tmp, g->stream, [&](void* t, size_t& b) {
    return cub::DeviceScan::InclusiveSum(t, b, d_main_row, d_main_row, (int)g->n_part, g->stream);
  }));
  uint64_t chk = 0;
  LUXB_CUDA(cudaMemcpyAsync(&chk, d_main_row + g->n_part - 1, 8, cudaMemcpyDeviceToHost, g->stream));
  LUXB_CUDA(cudaStreamSynchronize(g->stream));
  if (chk != e_main) { set_error("panel split: offsets do not add up"); return LUXB_ERR_STATE; }
  tmp.release(d_key2);
  tmp.release(d_pay2);
  LUXB_TRY(build_main_stream(g, d_main_row, d_main_src, e_main, d_hub_bits));
  tmp.release(d_main_row);
  tmp.release(d_main_src);

  // 7. raw sums of every slot: each sweep of the group streams writes all of them (pairs without edges have none)
  LUXB_TRY(gmalloc(g, &g->d_sb_partial, (uint64_t)n_slots + 1));
  g->d_hub_vtx = d_hub_vtx; tmp.keep(g, d_hub_vtx);
  g->d_hub_bits = d_hub_bits; tmp.keep(g, d_hub_bits);
  g->d_slot_bits = d_slot_bits; tmp.keep(g, d_slot_bits);
  g->d_slot_pre = d_slot_pre; tmp.keep(g, d_slot_pre);
  g->sb_n_hub = Nh;
  g->sb_n_blocks = NB;
  g->sb_n_groups = NG;
  g->sb_bs = bs;
  g->sb_on = true;
  g->cs_on = S > 0;
  const uint64_t NV = g->sb_groups.vbase[NB];
  g->stats.panel_edges = e_cov0;
  g->stats.panel_hubs = Nh;
  g->stats.panel_blocks = NB0;
  g->stats.cold_hub_edges = e_cold;
  g->stats.cold_hub_segments = S;
  g->stats.tier_blocks = NB - NB0;
  g->stats.tier_slots = NV - (uint64_t)NB0 * Nh;
  g->stats.tier_edges = e_cov - e_cov0;
  if (g->cfg.verbose) {
    printf("[luxb rank %d] source-blocked sweep: %u hub destinations (in-degree >= %u) x %u blocks of %u hot sources, + %u tier blocks "
           "(%llu slots, %llu edges); panel %llu edges (%.1f %%), cold-hub %llu edges (%u segments of %u values), main %llu edges\n",
           g->cfg.rank, Nh, st.sb_min_indeg, NB0, bs, NB - NB0, (unsigned long long)(NV - (uint64_t)NB0 * Nh), (unsigned long long)(e_cov - e_cov0),
           (unsigned long long)e_cov, 100.0 * e_cov / g->e_part, (unsigned long long)e_cold, S, cs.seg, (unsigned long long)e_main);
    printf("[luxb rank %d] (group, hub) pairs with edges / all: tier 0 %u / %llu, tiers %u / %llu, cold segments %u / %llu\n", g->cfg.rank,
           kind_slots[1], (unsigned long long)NB0 * Nh, kind_slots[2] - kind_slots[1], (unsigned long long)(NV - (uint64_t)NB0 * Nh),
           kind_slots[3] - kind_slots[2], (unsigned long long)Nh * S);
  }
  return 0;
}

// The pull sweep's structures (PageRank; CC / SSSP pull iterations): the flagged stream(s) of seg.cuh.
// LUXB_SWEEP=merge keeps the merge-path tiles of pull.cuh.
static int build_seg_sweep(luxb_graph* g) {
  g->seg_on = false;
  g->sb_on = false;
  if (!g->sweep.seg) return 0;
  if (g->n_part == 0 || g->cfg.zero_copy_edges || g->e_part >= 0xFFFFFFF0ull) return 0;  // zero-copy graphs keep the canonical arrays
  LUXB_TRY(build_panel_layout(g));
  if (!g->sb_on) LUXB_TRY(build_main_stream(g, g->d_row_end, g->hot_n ? g->d_src_gather : g->d_src, g->e_part, nullptr));
  g->seg_on = true;
  return 0;
}

extern "C++" {
// sms: the SMs whose worth of CTAs (ctas_per_sm each) the grid holds; st: the stream
template <class Prog, class Shape>
static int launch_seg_shape(luxb_graph* g, const SegArgs<Prog>& a, int sms, int ctas_per_sm, cudaStream_t st) {
  auto kern = seg_tile_kernel<Prog, Shape>;
  // The panel kernel holds one persistent CTA with ~all of the shared memory on every SM it runs on; when the cold half
  // of the exchange is in flight on the second stream (several ranks), a few SMs are left to NCCL's channel CTAs —
  // otherwise the collective could only start once the panel kernel has finished.
  const int reserve = (Shape::kPanel && g->packed) ? g->panel_reserve_sms : 0;
  LUXB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)Shape::kSmemBytes));
  int carve_pct = (int)std::min<size_t>(100, (ctas_per_sm * (Shape::kSmemBytes + 1024) * 100 + 228 * 1024 - 1) / (228 * 1024));
  LUXB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributePreferredSharedMemoryCarveout, carve_pct));
  const uint32_t grid = (uint32_t)std::min<uint64_t>((uint64_t)std::max(std::min(sms, g->num_sms - reserve), 1) * ctas_per_sm, a.n_stages);
  kern<<<grid, Shape::kThreads, Shape::kSmemBytes, st>>>(a);
  LUXB_CUDA(cudaGetLastError());
  return 0;
}

// the fields of a that come from the flagged stream L (seg.cuh); counter_slot: the stream's tile counter in d_counters
// (main 2, panel 4, cold-hub 5), which sweep_seg zeroes before the sweep.  The caller sets the stream-specific fields.
template <class Prog>
static void seg_stream_args(luxb_graph* g, PullLayout& L, SegArgs<Prog>& a, int counter_slot) {
  a.p.tile_v = L.d_tile_v;
  a.p.n_tiles = L.n_tiles;
  fill_fixup_args(a.p, L.fix);
  a.p.close_vtx = L.d_close;
  a.piece_slot = L.d_piece_slot;
  a.words = L.d_src;
  a.n_stages = L.n_stages;
  a.tile_counter = reinterpret_cast<uint32_t*>(g->d_counters + counter_slot);
}

// the seg kernel of one flagged stream in shape `shape` of the panel (kPanel) or the main family, on `sms` SMs' worth of
// CTAs, on stream st; its fix-up is the caller's.  kSlots: a main shape over a group stream (the cold-hub stream; the
// panel always is one).
template <bool kPanel, class Prog, bool kSlots = kPanel>
static int launch_seg_kernel(luxb_graph* g, const SegArgs<Prog>& a, int shape, int sms, int ctas_per_sm, cudaStream_t st,
                             const char* name) {
#define LUXB_CASE_MSHAPE(id, warps, stages, rounds) \
  case id: LUXB_TRY((launch_seg_shape<Prog, std::conditional_t<kSlots, SlotShape<SegMain##id>, SegMain##id>>(g, a, sms, ctas_per_sm, st))); break;
#define LUXB_CASE_PSHAPE(id, warps, stages, rounds, tab, v) \
  case id: LUXB_TRY((launch_seg_shape<Prog, SegPanel##id>(g, a, sms, ctas_per_sm, st))); break;
  if constexpr (kPanel) {
    switch (shape) {
      LUXB_SEG_PANEL_SHAPES(LUXB_CASE_PSHAPE)
      default: set_error("bad %s shape", name); return LUXB_ERR_STATE;
    }
  } else {
    switch (shape) {
      LUXB_SEG_MAIN_SHAPES(LUXB_CASE_MSHAPE)
      default: set_error("bad %s shape", name); return LUXB_ERR_STATE;
    }
  }
  g->stats.kernel_launches++;
  return 0;
}

// one flagged stream L swept on all SMs (g->stream), then its fix-up; tag: the phase-timer slot of the kernel
template <bool kPanel, class Prog, bool kSlots = kPanel>
static int launch_seg_stream(luxb_graph* g, PullLayout& L, const SegArgs<Prog>& a, int shape, int ctas_per_sm, int tag, const char* name) {
  LUXB_TRY((launch_seg_kernel<kPanel, Prog, kSlots>(g, a, shape, g->num_sms, ctas_per_sm, g->stream, name)));
  pt_mark(g, tag);
  return launch_fixup(g, a.p, L.fix, L.d_piece_slot);
}
}  // extern "C++"

extern "C++" {
// arguments of the main (L1) stream of a pull sweep
template <class Prog>
static SegArgs<Prog> seg_main_args(luxb_graph* g, PullLayout& L, const typename Prog::Vertex* x_nat, const typename Prog::Vertex* x_cold,
                                   typename Prog::Vertex* out_local, const typename Prog::Params& prm, const uint32_t* hub_bits) {
  SegArgs<Prog> a{};
  a.p.n_part = L.n_vtx;
  a.p.row_left = g->row_left;
  a.p.x_nat = x_nat;
  a.p.x_old = x_cold;
  a.p.x_hot = reinterpret_cast<const typename Prog::Vertex*>(g->d_hot);
  a.p.hot_n = g->hot_n;
  a.p.out = out_local;
  a.p.prm = prm;
  a.p.hub_bits = hub_bits;
  a.p.l2_hints = g->l2_hints;
  seg_stream_args(g, L, a, 2);
  return a;
}

// after the main stream's fix-up: its vertices without in-edges.
// out_buffer >= 0 (PageRank): index of the value buffer written, for the once-per-buffer constants of edge-less vertices;
// < 0 (labels): `out_local` already holds the old values, edge-less vertices keep them.
template <class Prog>
static int launch_seg_empties(luxb_graph* g, PullLayout& L, const PullArgs<Prog>& p, int out_buffer) {
  // PageRank: update(identity) is a constant -> written once per value buffer.  Hubs among them need the raw identity
  // every sweep (the combine overwrites it).
  if (out_buffer >= 0 && L.n_empty && !g->empties_done[out_buffer]) {
    empties_kernel<Prog><<<grid_for(L.n_empty, 256, g->num_sms * 8), 256, 0, g->stream>>>(p, L.d_empty, L.n_empty);
    g->empties_done[out_buffer] = true;
    g->stats.kernel_launches++;
  }
  if (L.n_empty_hub) {
    empties_kernel<Prog><<<grid_for(L.n_empty_hub, 256, g->num_sms * 8), 256, 0, g->stream>>>(p, L.d_empty_hub, L.n_empty_hub);
    g->stats.kernel_launches++;
  }
  LUXB_CUDA(cudaGetLastError());
  return 0;
}

// one pull sweep = [panel stream (shared-memory gathers) +] [cold-hub stream +] main stream (L1 gathers) [+ hub combine].
// The panel kernel is bound by shared-memory gathers and instruction issue on each SM; the cold-hub and main kernels
// by the rate at which the L2 serves random sector requests, a limit of the whole device rather than of each SM.  So
// on one rank (stream_b exists) with 0 < S = LUXB_PANEL_SMS < SMs they run at the same time:
//   g->stream:  panel kernel on S SMs -> panel fix-up -> main kernel again, S SMs' worth of CTAs ("join launch") -> join
//   stream_b:   cold-hub kernel on the other SMs -> cold-hub fix-up -> main kernel on the other SMs
// The two main launches share one SegArgs and so one tile counter: the join launch's CTAs claim whatever main stages
// are left once the panel is done, and every stage is still claimed exactly once, so the pieces, partials and fix-ups
// are those of the serial order and every value is bit for bit the same.  A panel CTA takes ~all of an SM's shared
// memory, so the side stream's CTAs cannot land on the panel's SMs while it runs; the panel is launched first so that
// its CTAs are dispatched before them.  Several ranks keep the serial order (stream2 carries the overlapped exchange).
template <class Prog>
static int sweep_seg(luxb_graph* g, const typename Prog::Vertex* x_nat, const typename Prog::Vertex* x_cold, typename Prog::Vertex* out_local,
                     int out_buffer, const typename Prog::Params& prm) {
  using Acc = typename Prog::Acc;
  constexpr bool kColdHub = std::is_same<Prog, PageRankProgram>::value;
  SegArgs<Prog> pa{}, ca{};
  if (g->sb_on) {
    pa.p.x_hot = reinterpret_cast<const typename Prog::Vertex*>(g->d_hot);
    pa.p.out = reinterpret_cast<typename Prog::Vertex*>(g->d_sb_partial);
    pa.p.raw_out = 1;
    pa.p.prm = prm;
    pa.bs = g->sb_bs;
    pa.n_blocks = g->sb_n_blocks;
    for (uint32_t b = 0; b < g->sb_n_blocks; ++b) pa.super_end[b] = g->sb_super_end[b];
    seg_stream_args(g, g->sb_panel, pa, 4);
  }
  if (g->cs_on) {
    // cold-hub stream: raw partial per (cold segment, hub) slot; its gathers all index the compact cold values, which it
    // loads with evict_normal (l2_hints = 0): the current segment is meant to stay in L2 while the SMs sweep it.  Only
    // PageRank builds it (the compact cold copy is PageRank's), so only PageRank instantiates its kernels.
    if constexpr (kColdHub) {
      ca.p.x_old = x_cold;
      ca.p.x_hot = reinterpret_cast<const typename Prog::Vertex*>(g->d_hot);
      ca.p.hot_n = g->hot_n;
      ca.p.out = reinterpret_cast<typename Prog::Vertex*>(g->d_sb_partial);
      ca.p.raw_out = 1;
      ca.p.l2_hints = 0;
      ca.p.prm = prm;
      seg_stream_args(g, g->sb_cold, ca, 5);
    } else {
      set_error("the cold-hub stream is built for PageRank only");
      return LUXB_ERR_STATE;
    }
  }
  const SegArgs<Prog> ma = seg_main_args<Prog>(g, g->sb_main, x_nat, x_cold, out_local, prm, g->sb_on ? g->d_hub_bits : nullptr);
  const int S = g->sweep.panel_sms;
  const bool beside = g->stream_b && S > 0 && S < g->num_sms;
  LUXB_TRY(kt_begin(g));
  LUXB_CUDA(cudaMemsetAsync(g->d_counters + 2, 0, 4, g->stream));
  if (g->sb_on) LUXB_CUDA(cudaMemsetAsync(g->d_counters + 4, 0, 16, g->stream));
  if (beside) {
    cudaStream_t sb = g->stream_b;
    LUXB_CUDA(cudaEventRecord(g->ev_fork, g->stream));
    const int t_fork = pt_event(g, g->stream);
    LUXB_TRY((launch_seg_kernel<true, Prog>(g, pa, g->sweep.panel_shape, S, 1, g->stream, "panel")));
    pt_mark(g, 5);
    LUXB_CUDA(cudaStreamWaitEvent(sb, g->ev_fork, 0));
    int t = pt_event(g, sb);
    if constexpr (kColdHub) {
      if (g->cs_on) {
        LUXB_TRY((launch_seg_kernel<false, Prog, true>(g, ca, g->sweep.cs_shape, g->num_sms - S, g->pull_ctas, sb, "cold-hub")));
        const int t_cold = pt_event(g, sb);
        pt_span(g, 9, t, t_cold);
        LUXB_TRY(launch_fixup(g, ca.p, g->sb_cold.fix, g->sb_cold.d_piece_slot, sb));
        t = pt_event(g, sb);
        pt_span(g, 1, t_cold, t);
      }
    }
    LUXB_TRY((launch_seg_kernel<false, Prog>(g, ma, g->sweep.main_shape, g->num_sms - S, g->pull_ctas, sb, "seg")));
    pt_span(g, 0, t, pt_event(g, sb));
    LUXB_CUDA(cudaEventRecord(g->ev_join, sb));
    LUXB_TRY(launch_fixup(g, pa.p, g->sb_panel.fix, g->sb_panel.d_piece_slot));
    pt_mark(g, 1);
    LUXB_TRY((launch_seg_kernel<false, Prog>(g, ma, g->sweep.main_shape, S, g->pull_ctas, g->stream, "seg")));
    pt_mark(g, 12);
    LUXB_CUDA(cudaStreamWaitEvent(g->stream, g->ev_join, 0));
    pt_mark(g, 13);
    pt_span(g, 14, t_fork, pt_event(g, g->stream));
  } else {
    if (g->sb_on) {
      LUXB_TRY((launch_seg_stream<true, Prog>(g, g->sb_panel, pa, g->sweep.panel_shape, 1, 5, "panel")));
      pt_mark(g, 1);
    }
    if constexpr (kColdHub) {
      if (g->cs_on) {
        LUXB_TRY((launch_seg_stream<false, Prog, true>(g, g->sb_cold, ca, g->sweep.cs_shape, g->pull_ctas, 9, "cold-hub")));
        pt_mark(g, 1);
      }
    }
    LUXB_TRY(wait_cold_exchange(g));
    LUXB_TRY((launch_seg_kernel<false, Prog>(g, ma, g->sweep.main_shape, g->num_sms, g->pull_ctas, g->stream, "seg")));
    pt_mark(g, 0);
  }
  LUXB_TRY(launch_fixup(g, ma.p, g->sb_main.fix, g->sb_main.d_piece_slot));
  LUXB_TRY(launch_seg_empties(g, g->sb_main, ma.p, out_buffer));
  pt_mark(g, 1);
  LUXB_TRY(kt_end(g));
  if (g->sb_on) {
    CombineArgs<Prog> cb{};
    cb.hub_vtx = g->d_hub_vtx;
    cb.n_hub = g->sb_n_hub;
    cb.n_blocks = g->sb_n_blocks;
    cb.n_groups = g->sb_n_groups;
    cb.row_left = g->row_left;
    cb.sg = g->sb_groups;
    cb.slot_bits = g->d_slot_bits;
    cb.slot_pre = g->d_slot_pre;
    cb.partial = reinterpret_cast<const Acc*>(g->d_sb_partial);
    cb.x_nat = x_nat;
    cb.out = out_local;
    cb.prm = prm;
    combine_hub_kernel<Prog><<<grid_for(g->sb_n_hub, 256, g->num_sms * 8), 256, 0, g->stream>>>(cb);
    LUXB_CUDA(cudaGetLastError());
    g->stats.kernel_launches++;
    pt_mark(g, 6);
  }
  return 0;
}
}  // extern "C++"

// After a sweep (or luxb_set_values): x_new holds this rank's final slice in natural order.  Make it visible to the
// next sweep of every rank: refresh the hot copies and, on several ranks, run the PACKED exchange — only vertices that are
// ever gathered travel (build.cuh), as one balanced all-gather written as kernels over peer memory: pack_push_kernel stores
// every owned entry into the transfer array of the rank holding its EQUAL chunk, a barrier (flag kernel) says the pushes
// have landed, chunk_pull_kernel copies the other ranks' chunks over NVLink.  Equal chunks because edge- or cost-balanced
// partitions own very different numbers of vertices (RMAT-27 at 8 GPUs: rank 7 owns 40 %): owner broadcasts or direct
// owner pushes (LUXB_PUSH=direct, measured 10 % slower at 4 GPUs) are bound by the biggest owner's egress.
static int pagerank_publish(luxb_graph* g, float* x_new) {
  const int me = g->cfg.rank;
  const int grid = g->num_sms * 8;
  if (g->P == 1 || !g->packed) {
    if (g->P > 1) { LUXB_TRY(allgather_slices(g, x_new, 4)); pt_mark(g, 3); }  // graphs without a hot set (tiny): plain all-gather
    if (g->hot_n) {
      const uint32_t z_n = g->hot_n + (g->cold_z ? g->cold_n : 0);
      hot_refresh_kernel<float><<<grid_for(z_n, 256, grid), 256, 0, g->stream>>>((float*)g->d_hot, x_new, g->d_hot_order, 0, z_n);
      LUXB_CUDA(cudaGetLastError());
      g->stats.kernel_launches++;
      pt_mark(g, 2);
    }
    return 0;
  }
  LUXB_TRY(wait_cold_exchange(g));  // back-to-back publishes (set_values after init): the buffer about to be packed is quiescent
  float* XTn = g->d_xt[1 - g->cur_xt];
  const uint32_t H = g->hot_n;
  const uint64_t Ch = g->xt_hot_chunk, Cc = g->xt_cold_chunk, cold_base = Ch * g->P;  // XT = [P hot chunks | P cold chunks]
  const uint32_t nh_me = g->hot_off[me + 1] - g->hot_off[me], nc_me = g->cold_off[me + 1] - g->cold_off[me];
  const bool p2p = g->p2p_ready && g->cfg.exchange != LUXB_EXCHANGE_NCCL;
  if (p2p) {
    // ---- balanced all-gather with three kernel launches and one 4-byte collective per iteration ----
    // 1. pack + push: every owned entry goes straight to the rank holding its equal chunk (remote stores);
    // 2. barrier: all pushes have landed;
    // 3. pull: every rank copies the chunks it does not hold from their holders (peer loads) — the hot region on the
    //    compute stream (the next sweep's panel gather needs it first), the cold region on the second stream,
    //    overlapped with that panel kernel (only the next MAIN sweep waits for it).
    if (nh_me + nc_me) {
      PackPushArgs<float> pa{};
      pa.x_local = x_new + g->row_left;
      pa.list = g->d_pack_list;
      pa.n_hot = nh_me;
      pa.n_cold = nc_me;
      pa.hot_pos0 = g->hot_off[me];
      pa.cold_pos0 = g->cold_off[me];
      pa.hot_chunk = Ch;
      pa.cold_chunk = Cc;
      pa.cold_base = cold_base;
      for (int k = 0; k < g->P; ++k) pa.xt[k] = reinterpret_cast<float*>(g->peer_xt[1 - g->cur_xt][k]);
      pa.P = g->P;
      const int pgrid = grid_for((uint64_t)nh_me + nc_me, 256, grid);
      if (g->direct_push) pack_push_kernel<float, true><<<pgrid, 256, 0, g->stream>>>(pa);
      else pack_push_kernel<float, false><<<pgrid, 256, 0, g->stream>>>(pa);
      LUXB_CUDA(cudaGetLastError());
      g->stats.kernel_launches++;
    }
    pt_mark(g, 7);
    LUXB_TRY(p2p_barrier(g));
    pt_mark(g, 4);
    auto pull = [&](uint64_t base, uint64_t C, cudaStream_t st, int ctas) -> int {
      ChunkPullArgs ca{};
      ca.dst = XTn + base;
      for (int k = 0; k < g->P; ++k) ca.src[k] = reinterpret_cast<const float*>(g->peer_xt[1 - g->cur_xt][k]) + base;
      ca.chunk = C;
      ca.P = g->P;
      ca.me = me;
      chunk_pull_kernel<<<ctas, 512, 0, st>>>(ca);
      LUXB_CUDA(cudaGetLastError());
      g->stats.kernel_launches++;
      return 0;
    };
    if (g->direct_push) {
      // everything is already in place: the owners stored into every rank's transfer array
    } else if (g->overlap_exchange) {
      LUXB_CUDA(cudaEventRecord(g->ev_pack, g->stream));  // = "barrier passed"
      LUXB_TRY(pull(0, Ch, g->stream, g->num_sms * 2));   // first in line: the next panel kernel waits for it
      LUXB_CUDA(cudaStreamWaitEvent(g->stream2, g->ev_pack, 0));
      // beside the panel kernel: only the SMs that kernel leaves free (launch_seg_shape)
      LUXB_TRY(pull(cold_base, Cc, g->stream2, std::max(2 * g->panel_reserve_sms, 8)));
      LUXB_CUDA(cudaEventRecord(g->ev_cold, g->stream2));
      g->cold_pending = true;
    } else {
      LUXB_TRY(pull(0, Ch, g->stream, g->num_sms * 2));
      LUXB_TRY(pull(cold_base, Cc, g->stream, g->num_sms * 2));
    }
    pt_mark(g, 8);
  } else {
    // NCCL only (no peer mappings): local pack, then one grouped set of in-place broadcasts per region
    if (nh_me + nc_me) {
      pack_values_kernel<float><<<grid_for((uint64_t)nh_me + nc_me, 256, grid), 256, 0, g->stream>>>(
          x_new + g->row_left, g->d_pack_list, nh_me, nc_me, XTn + g->hot_off[me], XTn + cold_base + g->cold_off[me]);
      LUXB_CUDA(cudaGetLastError());
      g->stats.kernel_launches++;
    }
    pt_mark(g, 7);
    LUXB_NCCL(nccl().GroupStart());
    for (int p = 0; p < g->P; ++p) {
      const uint32_t nh = g->hot_off[p + 1] - g->hot_off[p], nc = g->cold_off[p + 1] - g->cold_off[p];
      if (nh) LUXB_NCCL(nccl().Broadcast(XTn + g->hot_off[p], XTn + g->hot_off[p], nh, ncclFloat32, p, g->comm, g->stream));
      if (nc) LUXB_NCCL(nccl().Broadcast(XTn + cold_base + g->cold_off[p], XTn + cold_base + g->cold_off[p], nc, ncclFloat32, p, g->comm,
                                         g->stream));
    }
    LUXB_NCCL(nccl().GroupEnd());
    pt_mark(g, 8);
  }
  hot_permute_kernel<float><<<grid_for(H, 256, grid), 256, 0, g->stream>>>((float*)g->d_hot, XTn, g->d_zperm, H);
  LUXB_CUDA(cudaGetLastError());
  g->stats.kernel_launches++;
  pt_mark(g, 2);
  g->cur_xt ^= 1;
  g->replica_stale = true;
  return 0;
}

// the cold values of the previous exchange must have arrived before anything gathers them
static int wait_cold_exchange(luxb_graph* g) {
  if (g->cold_pending) {
    LUXB_CUDA(cudaStreamWaitEvent(g->stream, g->ev_cold, 0));
    g->cold_pending = false;
  }
  return 0;
}

static int pagerank_iteration(luxb_graph* g) {
  pt_mark(g, -1);
  PageRankProgram::Params prm;
  prm.init_rank = (1.0f - kAlpha) / (float)g->nv;  // pagerank_gpu.cu:144
  prm.deg = g->d_deg;
  float* x_old = (float*)g->d_val[g->cur];
  float* x_new = (float*)g->d_val[1 - g->cur];
  const float* x_cold = g->packed ? g->d_xt[g->cur_xt] + g->xt_hot_chunk * g->P : g->cold_z ? (const float*)g->d_hot + g->hot_n : x_old;
  if (g->seg_on) {
    LUXB_TRY((sweep_seg<PageRankProgram>(g, x_old, x_cold, x_new + g->row_left, 1 - g->cur, prm)));
  } else {
    LUXB_TRY(wait_cold_exchange(g));
    LUXB_TRY(launch_pull<PageRankProgram>(g, g->base, g->hot_n ? g->d_src_gather : g->d_src, x_old, x_cold, (const float*)g->d_hot,
                                          g->hot_n, x_new + g->row_left, prm));
  }
  LUXB_TRY(pagerank_publish(g, x_new));
  g->cur ^= 1;
  g->stats.edges_processed += g->e_part;
  return 0;
}

static int colfilter_iteration(luxb_graph* g) {
  float* x_old = (float*)g->d_val[g->cur];
  float* x_new = (float*)g->d_val[1 - g->cur];
  if (g->n_part) {
    CfArgs a{};
    a.row_end = g->d_row_end;
    a.src = g->d_src;
    a.weight = g->d_weight;
    a.chunk_first = g->cf.chunk_first;
    a.chunk_vtx = g->cf.chunk_vtx;
    a.n_part = g->n_part;
    a.n_chunks = g->cf.n_chunks;
    a.row_left = g->row_left;
    a.x_old = x_old;
    a.partial = g->cf.partial;
    a.out = x_new + (size_t)g->row_left * kCfK;
    a.n_peers = 0;
    if (g->p2p_ready && g->cfg.exchange != LUXB_EXCHANGE_NCCL)
      for (int p = 0; p < g->P; ++p)
        if (p != g->cfg.rank) a.peer_out[a.n_peers++] = (float*)g->peer_val[1 - g->cur][p] + (size_t)g->row_left * kCfK;
    uint64_t warps = g->cf.n_chunks;
    int grid = (int)std::min<uint64_t>((warps * 32 + 255) / 256, (uint64_t)g->num_sms * 8);
    cf_chunk_kernel<<<grid, 256, 0, g->stream>>>(a);
    cf_update_kernel<<<grid_for((uint64_t)g->n_part * kCfK, 256, g->num_sms * 8), 256, 0, g->stream>>>(a);
    LUXB_CUDA(cudaGetLastError());
    g->stats.kernel_launches += 2;
  }
  if (g->P > 1) {
    if (g->p2p_ready && g->cfg.exchange != LUXB_EXCHANGE_NCCL) LUXB_TRY(p2p_barrier(g));
    else LUXB_TRY(allgather_slices(g, x_new, 4 * kCfK));
  }
  g->cur ^= 1;
  g->stats.edges_processed += g->e_part;
  return 0;
}

// one PushAppTask (push_app_task_impl, components_gpu.cu:335-522) on this rank, including the exchange
extern "C++" {
template <class Prog>
static int label_iteration(luxb_graph* g) {
  const int me = g->cfg.rank;
  uint32_t* lab = reinterpret_cast<uint32_t*>(g->d_val[0]);
  // direction + representation decisions from the gathered headers (components_gpu.cu:397-416)
  uint64_t old_size = 0;
  int dense_parts = 0, sparse_parts = 0;
  for (int p = 0; p < g->P; ++p) {
    old_size += g->h_hdr[2 * p + 1];
    if (g->h_hdr[2 * p] == LUXB_DENSE_BITMAP) dense_parts++; else sparse_parts++;
  }
  bool dense_fq = dense_parts >= sparse_parts;
  const bool pull = old_size > (uint64_t)(g->nv / 16);
  if (pull) dense_fq = true;
  const uint32_t max_nodes = g->cap[me];
  unsigned char* new_slot = g->d_fq_new;
  LUXB_CUDA(cudaMemsetAsync(new_slot, 0, 8, g->stream));  // components_gpu.cu:412

  if (pull) {
    typename Prog::Params prm{0};
    if (g->hot_n) {
      hot_refresh_kernel<uint32_t><<<grid_for(g->hot_n, 256, g->num_sms * 8), 256, 0, g->stream>>>((uint32_t*)g->d_hot, lab, g->d_hot_order, 0, g->hot_n);
      g->stats.kernel_launches++;
    }
    bool swept = false;
    if constexpr (!Prog::kWeighted) {  // weighted programs never build the flagged streams (no weights there)
      if (g->seg_on) {
        LUXB_TRY((sweep_seg<Prog>(g, lab, lab, g->d_cur, -1, prm)));
        swept = true;
      }
    }
    if (!swept)
      LUXB_TRY(launch_pull<Prog>(g, g->base, g->hot_n ? g->d_src_gather : g->d_src, lab, lab, (const uint32_t*)g->d_hot, g->hot_n,
                                 g->d_cur, prm));
    g->stats.edges_processed += g->e_part;
    g->stats.pull_iterations++;
  } else if (g->n_part && old_size) {
    PushArgs a{};
    uint64_t blocks = 0;
    for (int p = 0; p < g->P; ++p) {
      a.fr[p].slot = slot_ptr(g->d_fq_all, g, p);
      a.fr[p].row_left = g->rl[p];
      a.fr[p].n_part = g->np[p];
      a.fr[p].type = g->h_hdr[2 * p];
      a.fr[p].count = std::min(g->h_hdr[2 * p + 1], g->cap[p]);
      uint32_t entries = a.fr[p].type == LUXB_DENSE_BITMAP ? (g->h_hdr[2 * p + 1] ? g->np[p] : 0) : a.fr[p].count;
      if (a.fr[p].type == LUXB_DENSE_BITMAP && g->h_hdr[2 * p + 1] == 0) a.fr[p].n_part = 0;
      blocks += (entries + kPushThreads - 1) / kPushThreads;
    }
    a.n_parts = g->P;
    a.out_end = g->d_out_end;
    a.out_dst = g->d_out_dst;
    a.lab = lab;
    a.cur = g->d_cur;
    a.row_left = g->row_left;
    a.new_sparse = dense_fq ? 0 : 1;
    a.new_count = reinterpret_cast<uint32_t*>(new_slot) + 1;
    a.new_queue = reinterpret_cast<uint32_t*>(new_slot + 8);
    a.max_nodes = max_nodes;
    a.edges_scanned = g->d_counters;
    a.big_list = reinterpret_cast<PushArgs::BigSeg*>(g->d_big_list);
    a.big_count = reinterpret_cast<uint32_t*>(g->d_counters + 3);
    a.big_capacity = g->big_capacity;
    a.out_w = g->d_out_w;
    if (blocks) {
      LUXB_CUDA(cudaMemsetAsync(a.big_count, 0, 4, g->stream));
      push_relax_kernel<Prog><<<(unsigned)blocks, kPushThreads, 0, g->stream>>>(a);
      push_big_kernel<Prog><<<g->num_sms * 4, kPushThreads, 0, g->stream>>>(a);
      LUXB_CUDA(cudaGetLastError());
      g->stats.kernel_launches += 2;
    }
  }

  const int fgrid = grid_for(g->n_part, 256, g->num_sms * 8);
  uint32_t count = 0;
  uint64_t total = 0;
  FrontierHeader my_hdr{LUXB_SPARSE_QUEUE, 0};
  const bool dev_frontier = g->P == 1 || (g->p2p_ready && g->cfg.exchange != LUXB_EXCHANGE_NCCL);
  if (dev_frontier) {
    // ---- new frontier + exchange WITHOUT host round trips: the representation rules (components_gpu.cu:462-491) run on
    // the device (push.cuh), the published slot and labels are stored straight into every rank's slot table / label
    // replica (frontier P2P push), and the host reads the P headers once, at the end of the iteration ----
    unsigned char* slot_d = dense_fq ? new_slot : g->d_fq_tmp;   // bitmap candidate
    unsigned char* slot_s = dense_fq ? g->d_fq_tmp : new_slot;   // queue candidate (filled by the push kernels)
    LUXB_CUDA(cudaMemsetAsync(dense_fq ? slot_s : slot_d, 0, 8, g->stream));
    if (!g->d_fctl) LUXB_TRY(gmalloc(g, &g->d_fctl, 1));
    if (dense_fq) frontier_diff_kernel<<<fgrid, 256, 0, g->stream>>>(lab + g->row_left, g->d_cur, g->n_part, slot_d);
    frontier_fix_kernel<<<1, 32, 0, g->stream>>>(slot_d, slot_s, max_nodes, dense_fq ? 1 : 0, g->d_fctl);
    frontier_d2s_if_kernel<<<fgrid, 256, 0, g->stream>>>(&g->d_fctl->need_d2s, slot_d, g->row_left, g->n_part, slot_s, max_nodes);
    frontier_diff_if_kernel<<<fgrid, 256, 0, g->stream>>>(&g->d_fctl->need_promote, lab + g->row_left, g->d_cur, g->n_part, slot_d);
    frontier_final_kernel<<<1, 32, 0, g->stream>>>(slot_d, slot_s, dense_fq ? 1 : 0, g->d_fctl);
    frontier_pack_labels_if_kernel<<<grid_for(max_nodes, 256, g->num_sms * 4), 256, 0, g->stream>>>(&g->d_fctl->final_sparse, slot_s, max_nodes,
                                                                                                  g->row_left, g->d_cur);
    LUXB_CUDA(cudaGetLastError());
    g->stats.kernel_launches += dense_fq ? 6 : 5;
    // barrier: every rank has finished the kernels that read this iteration's slots and labels
    if (g->P > 1) LUXB_TRY(p2p_barrier(g));
    FrontierPushArgs fa{};
    fa.ctl = g->d_fctl;
    fa.slot_d = slot_d;
    fa.slot_s = slot_s;
    fa.cur = g->d_cur;
    fa.n_part = g->n_part;
    fa.cap = g->cap[me];
    fa.row_left = g->row_left;
    fa.n_dst = 0;
    for (int p = 0; p < g->P; ++p) {
      unsigned char* fq_p = (p == me) ? g->d_fq_all : reinterpret_cast<unsigned char*>(g->peer_fq[p]);
      uint32_t* lab_p = (p == me) ? lab : reinterpret_cast<uint32_t*>(g->peer_val[0][p]);
      fa.dst_slot[fa.n_dst] = fq_p + g->slot_off[me];
      fa.dst_lab[fa.n_dst] = lab_p;
      fa.n_dst++;
    }
    frontier_push_kernel<<<g->num_sms * 2, 512, 0, g->stream>>>(fa);
    LUXB_CUDA(cudaGetLastError());
    g->stats.kernel_launches++;
    if (g->P > 1) LUXB_TRY(p2p_barrier(g));  // all pushes have landed
    PartTable pt{};
    pt.P = g->P;
    if (!g->d_slot_off) {
      LUXB_TRY(gmalloc(g, &g->d_slot_off, LUXB_MAX_PARTS));
      LUXB_CUDA(cudaMemcpyAsync(g->d_slot_off, g->slot_off, sizeof(uint64_t) * g->P, cudaMemcpyHostToDevice, g->stream));
    }
    frontier_headers_kernel<<<1, LUXB_MAX_PARTS, 0, g->stream>>>(g->d_fq_all, pt, g->d_slot_off, g->d_hdr_all);
    LUXB_CUDA(cudaMemcpyAsync(g->h_hdr, g->d_hdr_all, (size_t)g->P * 8, cudaMemcpyDeviceToHost, g->stream));
    LUXB_CUDA(cudaStreamSynchronize(g->stream));  // the iteration's one host synchronisation
    my_hdr.type = g->h_hdr[2 * me];
    my_hdr.num_nodes = count = g->h_hdr[2 * me + 1];
    for (int p = 0; p < g->P; ++p) total += g->h_hdr[2 * p + 1];
  } else {
    // ---- new frontier of this partition (components_gpu.cu:462-491) ----
    if (dense_fq) {
      if (g->n_part) {
        frontier_diff_kernel<<<fgrid, 256, 0, g->stream>>>(lab + g->row_left, g->d_cur, g->n_part, new_slot);
        g->stats.kernel_launches++;
      }
      LUXB_CUDA(cudaMemcpyAsync(g->h_scratch, new_slot, 8, cudaMemcpyDeviceToHost, g->stream));
      LUXB_CUDA(cudaStreamSynchronize(g->stream));
      count = g->h_scratch[1];
      if (count < max_nodes) {  // demote to a queue
        LUXB_CUDA(cudaMemsetAsync(g->d_fq_tmp, 0, 8, g->stream));
        if (count) {
          frontier_d2s_kernel<<<fgrid, 256, 0, g->stream>>>(new_slot, g->row_left, g->n_part, g->d_fq_tmp, max_nodes);
          g->stats.kernel_launches++;
        }
        std::swap(g->d_fq_new, g->d_fq_tmp);
        new_slot = g->d_fq_new;
        dense_fq = false;
      }
    } else {
      LUXB_CUDA(cudaMemcpyAsync(g->h_scratch, new_slot, 8, cudaMemcpyDeviceToHost, g->stream));
      LUXB_CUDA(cudaStreamSynchronize(g->stream));
      count = g->h_scratch[1];
      if (count >= max_nodes) {  // promote: rebuild as a bitmap from the label diff (count is re-derived exactly)
        dense_fq = true;
        LUXB_CUDA(cudaMemsetAsync(new_slot, 0, 8, g->stream));
        frontier_diff_kernel<<<fgrid, 256, 0, g->stream>>>(lab + g->row_left, g->d_cur, g->n_part, new_slot);
        g->stats.kernel_launches++;
        LUXB_CUDA(cudaMemcpyAsync(g->h_scratch, new_slot, 8, cudaMemcpyDeviceToHost, g->stream));
        LUXB_CUDA(cudaStreamSynchronize(g->stream));
        count = g->h_scratch[1];
      }
    }
    my_hdr = FrontierHeader{dense_fq ? LUXB_DENSE_BITMAP : LUXB_SPARSE_QUEUE, count};
    LUXB_CUDA(cudaMemcpyAsync(new_slot, &my_hdr, 8, cudaMemcpyHostToDevice, g->stream));
    if (!dense_fq && count) {
      frontier_pack_labels_kernel<<<grid_for(count, 256, g->num_sms * 4), 256, 0, g->stream>>>(new_slot, max_nodes, g->row_left,
                                                                                              g->d_cur);
      g->stats.kernel_launches++;
    }
    LUXB_CUDA(cudaGetLastError());

    // ---- exchange: headers, then payload sized by each partition's representation ----
    if (g->P > 1) {
      LUXB_NCCL(nccl().AllGather(new_slot, g->d_hdr_all, 8, ncclUint8, g->comm, g->stream));
      LUXB_CUDA(cudaMemcpyAsync(g->h_hdr, g->d_hdr_all, (size_t)g->P * 8, cudaMemcpyDeviceToHost, g->stream));
      LUXB_CUDA(cudaStreamSynchronize(g->stream));
    } else {
      g->h_hdr[0] = my_hdr.type;
      g->h_hdr[1] = my_hdr.num_nodes;
    }
    for (int p = 0; p < g->P; ++p) total += g->h_hdr[2 * p + 1];
    if (g->P > 1) {
      LUXB_NCCL(nccl().GroupStart());
      for (int p = 0; p < g->P; ++p) {
        uint32_t type = g->h_hdr[2 * p], cnt = g->h_hdr[2 * p + 1];
        unsigned char* dst_slot = slot_ptr(g->d_fq_all, g, p);
        const unsigned char* send_slot = p == me ? new_slot : dst_slot;
        LUXB_NCCL(nccl().Broadcast(send_slot, dst_slot, 8, ncclUint8, p, g->comm, g->stream));
        if (cnt == 0 || g->np[p] == 0) continue;
        if (type == LUXB_DENSE_BITMAP) {
          size_t bm_bytes = (((size_t)g->np[p] + 31) / 32) * 4;
          LUXB_NCCL(nccl().Broadcast(send_slot + 8, dst_slot + 8, bm_bytes, ncclUint8, p, g->comm, g->stream));
          const void* send_lab = p == me ? (const void*)g->d_cur : (const void*)(lab + g->rl[p]);
          LUXB_NCCL(nccl().Broadcast(send_lab, lab + g->rl[p], (size_t)g->np[p] * 4, ncclUint8, p, g->comm, g->stream));
        } else {
          size_t qoff = 8 + (size_t)g->cap[p] * 4;
          LUXB_NCCL(nccl().Broadcast(send_slot + 8, dst_slot + 8, (size_t)cnt * 4, ncclUint8, p, g->comm, g->stream));
          LUXB_NCCL(nccl().Broadcast(send_slot + qoff, dst_slot + qoff, (size_t)cnt * 4, ncclUint8, p, g->comm, g->stream));
        }
      }
      LUXB_NCCL(nccl().GroupEnd());
    } else {
      LUXB_CUDA(cudaMemcpyAsync(g->d_fq_all, new_slot, g->slot_bytes[0], cudaMemcpyDeviceToDevice, g->stream));
      if (dense_fq && count && g->n_part)
        LUXB_CUDA(cudaMemcpyAsync(lab + g->row_left, g->d_cur, (size_t)g->n_part * 4, cudaMemcpyDeviceToDevice, g->stream));
    }
  }
  for (int p = 0; p < g->P; ++p) {
    uint32_t type = g->h_hdr[2 * p], cnt = g->h_hdr[2 * p + 1];
    if (type == LUXB_SPARSE_QUEUE && cnt) {
      frontier_apply_kernel<<<grid_for(cnt, 256, g->num_sms * 4), 256, 0, g->stream>>>(slot_ptr(g->d_fq_all, g, p), g->cap[p], cnt, lab);
      g->stats.kernel_launches++;
    }
  }
  LUXB_CUDA(cudaGetLastError());
  g->stats.last_active = total;
  g->stats.last_frontier_type = my_hdr.type;
  g->trace_active.push_back(total);
  g->trace_pull.push_back(pull ? 1 : 0);
  if (g->cfg.verbose)
    printf("rowLeft(%u) activeNodes(%u) globalActive(%llu) %s\n", g->row_left, count, (unsigned long long)total, pull ? "pull" : "push");
  return 0;
}

}  // extern "C++"

static int one_iteration(luxb_graph* g) {
  switch (g->cfg.app) {
    case LUXB_PAGERANK: return pagerank_iteration(g);
    case LUXB_COLFILTER: return colfilter_iteration(g);
    case LUXB_CC: return label_iteration<MaxLabelProgram>(g);
    case LUXB_SSSP: return label_iteration<HopDistProgram>(g);
    case LUXB_SSSP_WEIGHTED: return label_iteration<WeightedDistProgram>(g);
  }
  return LUXB_ERR_ARG;
}

static int finish_timed(luxb_graph* g) {
  LUXB_TRY(wait_cold_exchange(g));  // the loop time includes the overlapped part of the last exchange
  pt_flush(g);
  if (g->pt.per_call) {  // LUXB_PHASE_TIMING=2: one line per luxb_iterate call instead of one per handle
    pt_print(g);
    for (double& v : g->pt.sum) v = 0;
    g->pt.chain = 0;
    g->pt.cnt = 0;
  }
  LUXB_CUDA(cudaEventRecord(g->ev_end, g->stream));
  LUXB_CUDA(cudaStreamSynchronize(g->stream));
  float ms = 0.f;
  LUXB_CUDA(cudaEventElapsedTime(&ms, g->ev_begin, g->ev_end));
  g->stats.loop_seconds += ms * 1e-3;
  if (g->h_barrier_err && *g->h_barrier_err) {
    set_error("iteration barrier: rank %u did not arrive within %llu s (LUXB_BARRIER_TIMEOUT_S)", *g->h_barrier_err - 1u,
              (unsigned long long)(g->barrier_timeout_ns / 1000000000ull));
    return LUXB_ERR_STATE;
  }
  for (size_t k = 0; k + 1 < g->kt_used; k += 2) {
    float kms = 0.f;
    LUXB_CUDA(cudaEventElapsedTime(&kms, g->kt_events[k], g->kt_events[k + 1]));
    g->stats.dominant_kernel_seconds += kms * 1e-3;
    g->stats.dominant_kernel_launches++;
  }
  g->kt_used = 0;
  if (g->d_out_end) {
    unsigned long long scanned = 0;
    LUXB_CUDA(cudaMemcpy(&scanned, g->d_counters, 8, cudaMemcpyDeviceToHost));
    LUXB_CUDA(cudaMemset(g->d_counters, 0, 8));
    g->stats.edges_processed += scanned;
  }
  return 0;
}

int luxb_iterate(luxb_graph* g, int iters, uint64_t* active_out) {
  LUXB_ARG(g != nullptr, "graph is NULL");
  if (!g->inited) { set_error("luxb_iterate before luxb_init"); return LUXB_ERR_STATE; }
  const AppInfo& app = app_of(g);
  LUXB_ARG(app.run != AppRun::kEntry, "luxb_iterate: %s runs through %s", app.name, app.entry);
  LUXB_ARG(iters >= 0, "negative iteration count");
  LUXB_CUDA(cudaSetDevice(g->cfg.device));
  if (const char* env = getenv("LUXB_PHASE_TIMING")) { g->pt.on = atoi(env) != 0; g->pt.per_call = atoi(env) == 2; }  // may change between calls
  LUXB_CUDA(cudaEventRecord(g->ev_begin, g->stream));
  for (int i = 0; i < iters; ++i) {
    LUXB_TRY(one_iteration(g));
    g->stats.iterations++;
  }
  LUXB_TRY(finish_timed(g));
  if (active_out) *active_out = g->stats.last_active;
  return 0;
}

int luxb_run_to_convergence(luxb_graph* g, int max_iters, int* iters_out) {
  LUXB_ARG(g != nullptr, "graph is NULL");
  if (!g->inited) { set_error("luxb_run_to_convergence before luxb_init"); return LUXB_ERR_STATE; }
  const AppInfo& app = app_of(g);
  LUXB_ARG(app.run != AppRun::kEntry, "luxb_run_to_convergence: %s runs through %s", app.name, app.entry);
  LUXB_ARG(app.run == AppRun::kConvergence, "only push apps converge (pagerank/col_filter run -ni iterations)");
  LUXB_CUDA(cudaSetDevice(g->cfg.device));
  LUXB_CUDA(cudaEventRecord(g->ev_begin, g->stream));
  int it = 0;
  while (max_iters <= 0 || it < max_iters) {
    LUXB_TRY(one_iteration(g));
    g->stats.iterations++;
    ++it;
    if (g->stats.last_active == 0) break;  // components.cc:116-123 without the 4-deep window
  }
  LUXB_TRY(finish_timed(g));
  if (iters_out) *iters_out = it;
  return 0;
}

// ---- betweenness centrality (bc.cuh) -------------------------------------------------------------------------------
extern "C++" {
// grow a device buffer to at least `need` elements (contents are not kept)
template <class T>
static int bc_grow(luxb_graph* g, T** p, uint64_t& cap, uint64_t need) {
  if (need <= cap) return 0;
  if (*p) { LUXB_TRY(gfree(g, *p)); *p = nullptr; cap = 0; }
  const uint64_t c = std::max<uint64_t>(need, 1024);
  LUXB_TRY(gmalloc(g, p, c));
  cap = c;
  return 0;
}
}  // extern "C++"

// σ, δ, scores (f64 x nv), the level order (u32 x nv), the sort's temporary storage and the hub segment tables (sized
// for this rank's edges: a vertex cut into segments has more than kBcSegment of them); the level buffers grow on demand
static int bc_alloc(luxb_graph* g) {
  LUXB_TRY(gmalloc(g, &g->bc.sigma, g->nv));
  LUXB_TRY(gmalloc(g, &g->bc.delta, g->nv));
  LUXB_TRY(gmalloc(g, &g->bc.scores, g->nv));
  LUXB_TRY(gmalloc(g, &g->bc.order, g->nv));
  LUXB_CUDA(cudaMemsetAsync(g->bc.scores, 0, (size_t)g->nv * 8, g->stream));
  cub::DoubleBuffer<uint32_t> keys(nullptr, nullptr), vals(nullptr, nullptr);
  LUXB_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, g->bc.sort_bytes, keys, vals, (int)g->nv, 0, 32, g->stream));
  if (g->cfg.app == LUXB_BC_WEIGHTED) {  // the class heads are selected with the same temporary storage after the sort
    size_t sel = 0;
    LUXB_CUDA(cub::DeviceSelect::If(nullptr, sel, thrust::counting_iterator<uint32_t>(0), (uint32_t*)nullptr, (uint32_t*)nullptr,
                                    (int)g->nv, BcClassHead{nullptr}, g->stream));
    g->bc.sort_bytes = std::max(g->bc.sort_bytes, sel);
  }
  LUXB_TRY(gmalloc(g, (char**)&g->bc.sort_tmp, g->bc.sort_bytes));
  LUXB_TRY(gmalloc(g, &g->bc.ctl, 5));
  LUXB_TRY(gmalloc(g, &g->bc.hubs, g->e_part / kBcSegment + 1));
  LUXB_TRY(gmalloc(g, &g->bc.partial, 2 * (g->e_part / kBcSegment) + 2));
  LUXB_CUDA(cudaStreamSynchronize(g->stream));
  return 0;
}

extern "C++" {
// the sum of f(neighbour) over the edge lists of n level vertices into out[0, n): main sweep, hub segments, combine.
// Hop levels keep the neighbours on level `target`; distance classes keep the tight edges
template <bool kOut>
static int bc_level_sum(luxb_graph* g, const uint32_t* order, uint32_t n, uint32_t target, double* out) {
  if (n == 0) return 0;
  BcLevelArgs a{};
  a.order = order;
  a.n = n;
  a.row_left = g->row_left;
  a.end = kOut ? g->d_out_end : g->d_row_end;
  a.nbr = kOut ? g->d_out_dst : g->d_src;
  a.lev = reinterpret_cast<const uint32_t*>(g->d_val[0]);
  a.target = target;
  a.sigma = g->bc.sigma;
  a.delta = g->bc.delta;
  a.out = out;
  a.ctl = reinterpret_cast<BcCtl*>(g->bc.ctl);
  a.hubs = g->bc.hubs;
  a.partial = g->bc.partial;
  a.edges = g->d_counters;
  LUXB_CUDA(cudaMemsetAsync(a.ctl, 0, sizeof(BcCtl), g->stream));
  const int grid = grid_for(n, kBcThreads / 32, g->num_sms * 16);
  if (g->cfg.app == LUXB_BC_WEIGHTED) {  // distance classes: tight edges at each vertex's own distance, target unused
    const BcClassArgs c{a, kOut ? g->d_out_w : g->d_weight};
    bc_class_sum_kernel<kOut><<<grid, kBcThreads, 0, g->stream>>>(c);
    bc_class_hub_segments_kernel<kOut><<<g->num_sms * 2, kBcThreads, 0, g->stream>>>(c);
  } else {
    bc_level_sum_kernel<kOut><<<grid, kBcThreads, 0, g->stream>>>(a);
    bc_hub_segments_kernel<kOut><<<g->num_sms * 2, kBcThreads, 0, g->stream>>>(a);
  }
  bc_combine_kernel<<<8, 128, 0, g->stream>>>(a.ctl, a.hubs, a.partial, out);
  LUXB_CUDA(cudaGetLastError());
  g->stats.kernel_launches += 3;
  return 0;
}
}  // extern "C++"

// nranks > 1: every partition's piece of each of the n_lists lists of bc.order delimited by bc.off, into bc.split
// and its host copy bc.h_split (read once the stream has synchronised)
static int bc_split(luxb_graph* g, uint32_t n_lists) {
  const uint32_t nv = g->nv;
  const uint64_t n = (uint64_t)n_lists * (g->P + 1);
  LUXB_TRY(bc_grow(g, &g->bc.split, g->bc.split_cap, n));
  BcSplitArgs sa{};
  for (int p = 0; p < g->P; ++p) sa.rl[p] = g->np[p] ? g->rl[p] : nv;
  sa.rl[g->P] = nv;
  for (int p = g->P - 1; p >= 0; --p) sa.rl[p] = std::min(sa.rl[p], sa.rl[p + 1]);
  sa.P = g->P;
  bc_split_kernel<<<grid_for(n, 256, g->num_sms * 8), 256, 0, g->stream>>>(g->bc.order, g->bc.off, n_lists, sa, g->bc.split);
  LUXB_CUDA(cudaGetLastError());
  g->bc.h_split.resize(n);
  LUXB_CUDA(cudaMemcpyAsync(g->bc.h_split.data(), g->bc.split, n * 4, cudaMemcpyDeviceToHost, g->stream));
  return 0;
}

// the level lists of the labels in the replica: order[], level_off (host bc_off, L + 1 entries) and, on several ranks,
// every partition's piece of every level (host bc_split)
static int bc_levels(luxb_graph* g, uint32_t& L) {
  const uint32_t nv = g->nv;
  const uint32_t* lev = reinterpret_cast<const uint32_t*>(g->d_val[0]);
  const int grid = g->num_sms * 8;
  LUXB_CUDA(cudaMemsetAsync(g->bc.ctl + 2, 0, 4, g->stream));
  bc_max_level_kernel<<<grid, 256, 0, g->stream>>>(lev, nv, g->bc.ctl + 2);
  uint32_t max_lev = 0;
  LUXB_CUDA(cudaMemcpyAsync(&max_lev, g->bc.ctl + 2, 4, cudaMemcpyDeviceToHost, g->stream));
  LUXB_CUDA(cudaStreamSynchronize(g->stream));
  L = max_lev + 1;
  int bits = 1;  // keys 0 .. L (L = unreached)
  while ((1ull << bits) <= L) ++bits;
  // σ and δ are free until the sweeps: they hold the sort's double buffers
  uint32_t* k0 = reinterpret_cast<uint32_t*>(g->bc.delta);
  uint32_t* v0 = reinterpret_cast<uint32_t*>(g->bc.sigma);
  bc_keys_kernel<<<grid, 256, 0, g->stream>>>(lev, nv, L, k0, v0);
  cub::DoubleBuffer<uint32_t> keys(k0, k0 + nv), vals(v0, g->bc.order);
  size_t bytes = g->bc.sort_bytes;
  LUXB_CUDA(cub::DeviceRadixSort::SortPairs(g->bc.sort_tmp, bytes, keys, vals, (int)nv, 0, bits, g->stream));
  if (vals.Current() != g->bc.order)
    LUXB_CUDA(cudaMemcpyAsync(g->bc.order, vals.Current(), (size_t)nv * 4, cudaMemcpyDeviceToDevice, g->stream));
  LUXB_TRY(bc_grow(g, &g->bc.off, g->bc.off_cap, (uint64_t)L + 1));
  fill_kernel<uint32_t><<<1, 32, 0, g->stream>>>(g->bc.off + L, 1, nv);
  bc_level_off_kernel<<<grid, 256, 0, g->stream>>>(keys.Current(), nv, g->bc.off);
  LUXB_CUDA(cudaGetLastError());
  g->bc.h_off.resize((size_t)L + 1);
  LUXB_CUDA(cudaMemcpyAsync(g->bc.h_off.data(), g->bc.off, ((size_t)L + 1) * 4, cudaMemcpyDeviceToHost, g->stream));
  if (g->P > 1) LUXB_TRY(bc_split(g, L));
  LUXB_CUDA(cudaStreamSynchronize(g->stream));
  g->stats.kernel_launches += g->P > 1 ? 6 : 5;
  return 0;
}

// the distance classes of the weighted distances in the replica: order[] sorted stably by distance, class_off (host
// bc_off, C + 1 entries, one class per distinct distance) and, on several ranks, every partition's piece of every class.
// The keys are sparse, so the class offsets are the positions where the sorted key changes.  The class count is only
// known on the device: the host reads a bound on it (min(reached, largest distance + 1)) worth of offsets, padded with
// empty classes, together with the count in one synchronisation.
static int bc_classes(luxb_graph* g, uint32_t& C) {
  const uint32_t nv = g->nv;
  const uint32_t* dist = reinterpret_cast<const uint32_t*>(g->d_val[0]);
  const int grid = g->num_sms * 8;
  uint32_t* ctl = g->bc.ctl;
  LUXB_CUDA(cudaMemsetAsync(ctl + 2, 0, 8, g->stream));
  bc_dist_max_kernel<<<grid, 256, 0, g->stream>>>(dist, nv, ctl + 2);
  uint32_t h[2] = {0, 0};
  LUXB_CUDA(cudaMemcpyAsync(h, ctl + 2, 8, cudaMemcpyDeviceToHost, g->stream));
  LUXB_CUDA(cudaStreamSynchronize(g->stream));
  const uint32_t reached = h[1], K = h[0] + 1;  // K: the key of the unreached (<= 2^32 - 1: a distance is < INF)
  int bits = 1;  // keys 0 .. K
  while ((1ull << bits) <= K) ++bits;
  uint32_t* k0 = reinterpret_cast<uint32_t*>(g->bc.delta);
  uint32_t* v0 = reinterpret_cast<uint32_t*>(g->bc.sigma);
  bc_dist_keys_kernel<<<grid, 256, 0, g->stream>>>(dist, nv, K, k0, v0);
  cub::DoubleBuffer<uint32_t> keys(k0, k0 + nv), vals(v0, g->bc.order);
  size_t bytes = g->bc.sort_bytes;
  LUXB_CUDA(cub::DeviceRadixSort::SortPairs(g->bc.sort_tmp, bytes, keys, vals, (int)nv, 0, bits, g->stream));
  if (vals.Current() != g->bc.order)
    LUXB_CUDA(cudaMemcpyAsync(g->bc.order, vals.Current(), (size_t)nv * 4, cudaMemcpyDeviceToDevice, g->stream));
  const uint32_t bound = (uint32_t)std::min<uint64_t>(reached, K);
  LUXB_TRY(bc_grow(g, &g->bc.off, g->bc.off_cap, (uint64_t)bound + 1));
  bytes = g->bc.sort_bytes;
  LUXB_CUDA(cub::DeviceSelect::If(g->bc.sort_tmp, bytes, thrust::counting_iterator<uint32_t>(0), g->bc.off, ctl + 4, (int)reached,
                                  BcClassHead{keys.Current()}, g->stream));
  bc_class_tail_kernel<<<grid_for((uint64_t)bound + 1, 256, grid), 256, 0, g->stream>>>(ctl + 4, bound + 1, reached, g->bc.off);
  LUXB_CUDA(cudaGetLastError());
  g->bc.h_off.resize((size_t)bound + 1);
  LUXB_CUDA(cudaMemcpyAsync(h, ctl + 4, 4, cudaMemcpyDeviceToHost, g->stream));
  LUXB_CUDA(cudaMemcpyAsync(g->bc.h_off.data(), g->bc.off, ((size_t)bound + 1) * 4, cudaMemcpyDeviceToHost, g->stream));
  if (g->P > 1) LUXB_TRY(bc_split(g, bound));
  LUXB_CUDA(cudaStreamSynchronize(g->stream));
  C = h[0];
  g->bc.h_off.resize((size_t)C + 1);
  g->stats.kernel_launches += g->P > 1 ? 6 : 5;
  return 0;
}

// one source: BFS levels or weighted distances (the SSSP engine), level / class lists, forward σ, backward δ,
// scores += δ.  Weighted, "level d" below is distance class d
static int bc_source(luxb_graph* g, uint32_t s) {
  const bool weighted = g->cfg.app == LUXB_BC_WEIGHTED;
  g->trace_active.clear();
  g->trace_pull.clear();
  LUXB_TRY(reset_label_state(g, false, s));
  do {
    LUXB_TRY(weighted ? label_iteration<WeightedDistProgram>(g) : label_iteration<HopDistProgram>(g));
    g->stats.iterations++;
  } while (g->stats.last_active != 0);
  uint32_t L = 0;
  LUXB_TRY(weighted ? bc_classes(g, L) : bc_levels(g, L));
  const std::vector<uint32_t>& off = g->bc.h_off;
  uint64_t widest = 0;
  for (uint32_t d = 0; d < L; ++d) widest = std::max<uint64_t>(widest, off[d + 1] - off[d]);
  LUXB_TRY(bc_grow(g, &g->bc.lvl, g->bc.lvl_cap, widest));
  LUXB_CUDA(cudaMemsetAsync(g->bc.sigma, 0, (size_t)g->nv * 8, g->stream));
  LUXB_CUDA(cudaMemsetAsync(g->bc.delta, 0, (size_t)g->nv * 8, g->stream));
  bc_source_kernel<<<1, 1, 0, g->stream>>>(g->bc.sigma, s);
  pt_mark(g, -1);
  const int me = g->cfg.rank, P1 = g->P + 1;
  const int grid = g->num_sms * 8;
  // forward: each rank sums σ for its own piece of level d over its CSC slice, the pieces are broadcast in place
  for (uint32_t d = 1; d < L; ++d) {
    const uint32_t o = off[d], n = off[d + 1] - o;
    const uint32_t a = g->P > 1 ? g->bc.h_split[(size_t)d * P1 + me] : o;
    const uint32_t b = g->P > 1 ? g->bc.h_split[(size_t)d * P1 + me + 1] : o + n;
    LUXB_TRY(bc_level_sum<false>(g, g->bc.order + a, b - a, d - 1, g->bc.lvl + (a - o)));
    if (g->P > 1) {
      LUXB_NCCL(nccl().GroupStart());
      for (int p = 0; p < g->P; ++p) {
        const uint32_t pa = g->bc.h_split[(size_t)d * P1 + p], pb = g->bc.h_split[(size_t)d * P1 + p + 1];
        if (pb == pa) continue;
        double* seg = g->bc.lvl + (pa - o);
        LUXB_NCCL(nccl().Broadcast(seg, seg, (size_t)(pb - pa) * 8, ncclUint8, p, g->comm, g->stream));
      }
      LUXB_NCCL(nccl().GroupEnd());
    }
    bc_sigma_finish_kernel<<<grid_for(n, 256, grid), 256, 0, g->stream>>>(g->bc.order + o, n, g->bc.lvl, g->bc.sigma);
    g->stats.kernel_launches++;
  }
  pt_mark(g, 10);
  // backward: every rank sums t over the out-edges that land in its partition for the whole level d - 1; the partial
  // sums are added across ranks in level order
  for (uint32_t d = L - 1; d >= 1; --d) {
    const uint32_t o = off[d - 1], n = off[d] - o;
    LUXB_TRY(bc_level_sum<true>(g, g->bc.order + o, n, d, g->bc.lvl));
    if (g->P > 1) LUXB_NCCL(nccl().AllReduce(g->bc.lvl, g->bc.lvl, n, ncclFloat64, ncclSum, g->comm, g->stream));
    bc_delta_finish_kernel<<<grid_for(n, 256, grid), 256, 0, g->stream>>>(g->bc.order + o, n, g->bc.lvl, g->bc.sigma, g->bc.delta);
    g->stats.kernel_launches++;
  }
  bc_accumulate_kernel<<<grid_for(off[L], 256, grid), 256, 0, g->stream>>>(g->bc.order, off[L], g->bc.delta, g->bc.scores);
  LUXB_CUDA(cudaGetLastError());
  g->stats.kernel_launches += 4;
  pt_mark(g, 11);
  g->bc.has_source = true;
  return 0;
}

int luxb_bc_run(luxb_graph* g, const luxb_vid* sources, int n_sources) {
  LUXB_ARG(g != nullptr, "graph is NULL");
  if (!g->inited) { set_error("luxb_bc_run before luxb_init"); return LUXB_ERR_STATE; }
  LUXB_ARG(app_of(g).entry == kBcRun, "luxb_bc_run needs a LUXB_BC or LUXB_BC_WEIGHTED handle (this one is app %d)", (int)g->cfg.app);
  LUXB_ARG(n_sources >= 0, "negative source count");
  LUXB_ARG(sources != nullptr || n_sources == 0, "sources is NULL");
  for (int i = 0; i < n_sources; ++i)
    LUXB_ARG(sources[i] < g->nv, "source %u (entry %d) >= nv (%u)", sources[i], i, g->nv);
  if (n_sources == 0) return 0;
  LUXB_CUDA(cudaSetDevice(g->cfg.device));
  if (const char* env = getenv("LUXB_PHASE_TIMING")) { g->pt.on = atoi(env) != 0; g->pt.per_call = atoi(env) == 2; }
  LUXB_CUDA(cudaEventRecord(g->ev_begin, g->stream));
  for (int i = 0; i < n_sources; ++i) LUXB_TRY(bc_source(g, sources[i]));
  return finish_timed(g);
}

int luxb_bc_source_state(luxb_graph* g, uint32_t* lev, double* sigma, double* delta, size_t nv_count) {
  LUXB_ARG(g != nullptr, "graph is NULL");
  if (!g->inited) { set_error("luxb_bc_source_state before luxb_init"); return LUXB_ERR_STATE; }
  LUXB_ARG(app_of(g).entry == kBcRun, "luxb_bc_source_state needs a LUXB_BC or LUXB_BC_WEIGHTED handle (this one is app %d)",
           (int)g->cfg.app);
  LUXB_ARG(nv_count == g->nv, "nv_count is %zu, the graph has %u vertices", nv_count, g->nv);
  if (!g->bc.has_source) { set_error("luxb_bc_source_state: no source processed yet"); return LUXB_ERR_STATE; }
  LUXB_CUDA(cudaSetDevice(g->cfg.device));
  if (lev) LUXB_CUDA(cudaMemcpyAsync(lev, g->d_val[0], (size_t)g->nv * 4, cudaMemcpyDeviceToHost, g->stream));
  if (sigma) LUXB_CUDA(cudaMemcpyAsync(sigma, g->bc.sigma, (size_t)g->nv * 8, cudaMemcpyDeviceToHost, g->stream));
  if (delta) LUXB_CUDA(cudaMemcpyAsync(delta, g->bc.delta, (size_t)g->nv * 8, cudaMemcpyDeviceToHost, g->stream));
  LUXB_CUDA(cudaStreamSynchronize(g->stream));
  return 0;
}

// ---- triangle counting (tc.cuh) ------------------------------------------------------------------------------------
// sort keys[0, n) over their low `bits` bits and keep the distinct ones, at the front of keys; *m = their number
static int tc_sort_unique(luxb_graph* g, DevTmp& tmp, uint64_t* keys, uint64_t* alt, uint64_t n, int bits, uint64_t* m) {
  *m = 0;
  if (n == 0) return 0;
  cub::DoubleBuffer<uint64_t> db(keys, alt);
  LUXB_TRY(cub_call(tmp, g->stream, [&](void* t, size_t& b) {
    return cub::DeviceRadixSort::SortKeys(t, b, db, (long long)n, 0, bits, g->stream);
  }));
  unsigned long long* d_n = nullptr;
  LUXB_TRY(tmp.alloc(&d_n, 1));
  uint64_t* out = db.Current() == keys ? alt : keys;
  LUXB_TRY(cub_call(tmp, g->stream, [&](void* t, size_t& b) {
    return cub::DeviceSelect::Unique(t, b, db.Current(), out, d_n, (long long)n, g->stream);
  }));
  unsigned long long cnt = 0;
  LUXB_CUDA(cudaMemcpyAsync(&cnt, d_n, 8, cudaMemcpyDeviceToHost, g->stream));
  LUXB_CUDA(cudaStreamSynchronize(g->stream));
  tmp.release(d_n);
  if (out != keys) LUXB_CUDA(cudaMemcpyAsync(keys, out, cnt * 8, cudaMemcpyDeviceToDevice, g->stream));
  *m = cnt;
  return 0;
}

// The distinct undirected keys min << 32 | max of the whole graph, on every rank (on several ranks every rank's distinct
// keys go to every rank), at the front of *keys; *alt is a buffer of the same size.  Both belong to `tmp`.  The graph of
// LUXB_TC, LUXB_KCORE and LUXB_TRUSS.
static int undirected_keys(luxb_graph* g, DevTmp& tmp, int bits, uint64_t** keys_out, uint64_t** alt_out, uint64_t* m_out) {
  const int grid = g->num_sms * 8;
  uint64_t *d_keys = nullptr, *d_alt = nullptr;
  unsigned long long* d_cur = nullptr;
  LUXB_TRY(tmp.alloc(&d_keys, g->e_part));
  LUXB_TRY(tmp.alloc(&d_alt, g->e_part));
  LUXB_TRY(tmp.alloc(&d_cur, 1));
  LUXB_CUDA(cudaMemsetAsync(d_cur, 0, 8, g->stream));
  if (g->e_part)
    tc_emit_keys_kernel<<<grid_for(g->e_part, 256, grid), 256, 0, g->stream>>>(g->d_row_end, g->n_part, g->e_part, g->row_left, g->d_src,
                                                                             d_cur, d_keys);
  LUXB_CUDA(cudaGetLastError());
  unsigned long long n_keys = 0;
  LUXB_CUDA(cudaMemcpyAsync(&n_keys, d_cur, 8, cudaMemcpyDeviceToHost, g->stream));
  LUXB_CUDA(cudaStreamSynchronize(g->stream));
  uint64_t m = 0;
  LUXB_TRY(tc_sort_unique(g, tmp, d_keys, d_alt, n_keys, bits, &m));
  if (g->P > 1) {  // every rank's distinct keys to every rank (one grouped set of broadcasts), distinct again
    uint64_t* d_counts = nullptr;
    LUXB_TRY(tmp.alloc(&d_counts, (uint64_t)g->P + 1));
    LUXB_CUDA(cudaMemcpyAsync(d_counts + g->P, &m, 8, cudaMemcpyHostToDevice, g->stream));
    LUXB_NCCL(nccl().AllGather(d_counts + g->P, d_counts, 1, ncclUint64, g->comm, g->stream));
    std::vector<uint64_t> counts(g->P);
    LUXB_CUDA(cudaMemcpyAsync(counts.data(), d_counts, (size_t)g->P * 8, cudaMemcpyDeviceToHost, g->stream));
    LUXB_CUDA(cudaStreamSynchronize(g->stream));
    uint64_t total = 0;
    for (uint64_t c : counts) total += c;
    uint64_t *d_all = nullptr, *d_all_alt = nullptr;
    LUXB_TRY(tmp.alloc(&d_all, total));
    LUXB_TRY(tmp.alloc(&d_all_alt, total));
    LUXB_NCCL(nccl().GroupStart());
    uint64_t at = 0;
    for (int p = 0; p < g->P; ++p) {
      if (counts[p]) LUXB_NCCL(nccl().Broadcast(p == g->cfg.rank ? d_keys : d_all + at, d_all + at, counts[p], ncclUint64, p, g->comm, g->stream));
      at += counts[p];
    }
    LUXB_NCCL(nccl().GroupEnd());
    LUXB_CUDA(cudaStreamSynchronize(g->stream));
    tmp.release(d_keys);
    tmp.release(d_alt);
    d_keys = d_all;
    d_alt = d_all_alt;
    LUXB_TRY(tc_sort_unique(g, tmp, d_keys, d_alt, total, bits, &m));
  }
  *keys_out = d_keys;
  *alt_out = d_alt;
  *m_out = m;
  return 0;
}

// bits of a sort key (high word) << 32 | (low word) over vertex ids < nv
static int pair_key_bits(uint32_t nv) {
  int vbits = 1;
  while ((1ull << vbits) < (uint64_t)nv) ++vbits;
  return 32 + vbits;
}

// The oriented out-lists of the m undirected keys (oriented in place, then released with `alt`), the work per vertex
// and the bins of this rank's range, into `tc` (off, dst, staged, stage_pre, group, n_group, big, n_big).  LUXB_TC and
// LUXB_TRUSS.
static int tc_orient_bins(luxb_graph* g, DevTmp& tmp, int bits, uint64_t* d_keys, uint64_t* d_alt, uint64_t m, TcState& tc) {
  const int grid = g->num_sms * 8;
  const uint32_t nv = g->nv;
  // degrees, orientation, out-lists sorted by (from, to), offsets and the work W(u)
  uint32_t *d_deg = nullptr, *d_outdeg = nullptr;
  unsigned long long* d_work = nullptr;
  LUXB_TRY(tmp.alloc(&d_deg, nv));
  LUXB_TRY(tmp.alloc(&d_outdeg, nv));
  LUXB_TRY(tmp.alloc(&d_work, nv));
  LUXB_CUDA(cudaMemsetAsync(d_deg, 0, (size_t)nv * 4, g->stream));
  LUXB_CUDA(cudaMemsetAsync(d_outdeg, 0, (size_t)nv * 4, g->stream));
  LUXB_CUDA(cudaMemsetAsync(d_work, 0, (size_t)nv * 8, g->stream));
  const uint64_t* d_sorted = d_keys;
  if (m) {
    tc_degree_kernel<<<grid_for(m, 256, grid), 256, 0, g->stream>>>(d_keys, m, d_deg);
    tc_orient_kernel<<<grid_for(m, 256, grid), 256, 0, g->stream>>>(d_keys, m, d_deg, d_outdeg);
    LUXB_CUDA(cudaGetLastError());
    cub::DoubleBuffer<uint64_t> db(d_keys, d_alt);
    LUXB_TRY(cub_call(tmp, g->stream, [&](void* t, size_t& b) {
      return cub::DeviceRadixSort::SortKeys(t, b, db, (long long)m, 0, bits, g->stream);
    }));
    d_sorted = db.Current();
  }
  LUXB_TRY(gmalloc(g, &tc.off, (uint64_t)nv + 1));
  LUXB_CUDA(cudaMemsetAsync(tc.off + nv, 0, 8, g->stream));
  widen_u32_to_u64_kernel<<<grid_for(nv, 256, grid), 256, 0, g->stream>>>(d_outdeg, tc.off, nv);
  LUXB_TRY(cub_call(tmp, g->stream, [&](void* t, size_t& b) {
    return cub::DeviceScan::ExclusiveSum(t, b, tc.off, tc.off, (long long)nv + 1, g->stream);
  }));
  LUXB_TRY(gmalloc(g, &tc.dst, m + 8));
  if (m) tc_lists_kernel<<<grid_for(m, 256, grid), 256, 0, g->stream>>>(d_sorted, m, tc.off, tc.dst, d_work);
  LUXB_CUDA(cudaGetLastError());
  LUXB_CUDA(cudaStreamSynchronize(g->stream));
  for (void* q : {(void*)d_keys, (void*)d_alt, (void*)d_deg, (void*)d_outdeg}) tmp.release(q);
  // bins of this rank's range: staged vertices (grouped kernel) and big ones
  uint32_t* d_sel = nullptr;
  LUXB_TRY(tmp.alloc(&d_sel, 2));
  LUXB_TRY(gmalloc(g, &tc.staged, g->n_part));
  LUXB_TRY(gmalloc(g, &tc.big, g->n_part));
  uint32_t n_sel[2] = {0, 0};
  if (g->n_part) {
    thrust::counting_iterator<uint32_t> ids(g->row_left);
    LUXB_TRY(cub_call(tmp, g->stream, [&](void* t, size_t& b) {
      return cub::DeviceSelect::If(t, b, ids, tc.staged, d_sel, (int)g->n_part, TcStaged{tc.off}, g->stream);
    }));
    LUXB_TRY(cub_call(tmp, g->stream, [&](void* t, size_t& b) {
      return cub::DeviceSelect::If(t, b, ids, tc.big, d_sel + 1, (int)g->n_part, TcBig{tc.off}, g->stream);
    }));
    LUXB_CUDA(cudaMemcpyAsync(n_sel, d_sel, 8, cudaMemcpyDeviceToHost, g->stream));
    LUXB_CUDA(cudaStreamSynchronize(g->stream));
  }
  const uint32_t n_staged = n_sel[0];
  tc.n_big = n_sel[1];
  // groups: exclusive prefixes of the staged list lengths and costs, a head wherever either crosses its multiple
  uint64_t* d_cost = nullptr;
  LUXB_TRY(tmp.alloc(&d_cost, (uint64_t)n_staged + 1));
  LUXB_TRY(gmalloc(g, &tc.stage_pre, (uint64_t)n_staged + 1));
  tc_cost_kernel<<<grid_for((uint64_t)n_staged + 1, 256, grid), 256, 0, g->stream>>>(tc.staged, n_staged, tc.off, d_work,
                                                                                    tc.stage_pre, d_cost);
  LUXB_CUDA(cudaGetLastError());
  for (uint64_t* p : {tc.stage_pre, d_cost})
    LUXB_TRY(cub_call(tmp, g->stream, [&](void* t, size_t& b) {
      return cub::DeviceScan::ExclusiveSum(t, b, p, p, (long long)n_staged + 1, g->stream);
    }));
  LUXB_TRY(gmalloc(g, &tc.group, (uint64_t)n_staged + 1));
  uint32_t n_group = 0;
  if (n_staged) {
    LUXB_TRY(cub_call(tmp, g->stream, [&](void* t, size_t& b) {
      return cub::DeviceSelect::If(t, b, thrust::counting_iterator<uint32_t>(0), tc.group, d_sel, (int)n_staged,
                                   TcGroupHead{tc.stage_pre, d_cost}, g->stream);
    }));
    LUXB_CUDA(cudaMemcpyAsync(&n_group, d_sel, 4, cudaMemcpyDeviceToHost, g->stream));
    LUXB_CUDA(cudaStreamSynchronize(g->stream));
  }
  LUXB_CUDA(cudaMemcpyAsync(tc.group + n_group, &n_staged, 4, cudaMemcpyHostToDevice, g->stream));
  tc.n_group = n_group;
  return 0;
}

// luxb_init of a LUXB_TC handle: the undirected simple edges of the whole graph (undirected_keys), the oriented
// out-lists, the work per vertex and the bins of this rank's range (tc_orient_bins)
static int tc_build(luxb_graph* g) {
  DevTmp tmp;
  const uint32_t nv = g->nv;
  const int bits = pair_key_bits(nv);  // min < nv in the high word, max in the low one
  uint64_t *d_keys = nullptr, *d_alt = nullptr;
  uint64_t m = 0;
  LUXB_TRY(undirected_keys(g, tmp, bits, &d_keys, &d_alt, &m));
  g->tc.m = m;
  LUXB_TRY(tc_orient_bins(g, tmp, bits, d_keys, d_alt, m, g->tc));
  // the run's state: t, its sum, the work counters; a grid of resident CTAs per kernel
  LUXB_TRY(gmalloc(g, &g->tc.t, nv));
  LUXB_CUDA(cudaMemsetAsync(g->tc.t, 0, (size_t)nv * 8, g->stream));
  LUXB_TRY(gmalloc(g, &g->tc.total, 1));
  LUXB_TRY(gmalloc(g, &g->tc.next, 2));
  LUXB_CUDA(cub::DeviceReduce::Sum(nullptr, g->tc.sum_bytes, g->tc.t, g->tc.total, (long long)nv, g->stream));
  LUXB_TRY(gmalloc(g, (char**)&g->tc.sum_tmp, g->tc.sum_bytes));
  int per_sm = 0;
  LUXB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, tc_group_kernel, kTcThreads, 0));
  g->tc.group_grid = std::max(per_sm, 1) * g->num_sms;
  LUXB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, tc_big_kernel, kTcThreads, 0));
  g->tc.big_grid = std::max(per_sm, 1) * g->num_sms;
  LUXB_CUDA(cudaStreamSynchronize(g->stream));
  return 0;
}

int luxb_tc_run(luxb_graph* g, uint64_t* total_out) {
  LUXB_ARG(g != nullptr, "graph is NULL");
  if (!g->inited) { set_error("luxb_tc_run before luxb_init"); return LUXB_ERR_STATE; }
  LUXB_ARG(g->cfg.app == LUXB_TC, "luxb_tc_run needs a LUXB_TC handle (this one is app %d)", (int)g->cfg.app);
  LUXB_CUDA(cudaSetDevice(g->cfg.device));
  LUXB_CUDA(cudaEventRecord(g->ev_begin, g->stream));
  LUXB_CUDA(cudaMemsetAsync(g->tc.t, 0, (size_t)g->nv * 8, g->stream));
  LUXB_CUDA(cudaMemsetAsync(g->tc.next, 0, 8, g->stream));
  const TcArgs a{g->tc.off, g->tc.dst, g->tc.staged, g->tc.stage_pre, g->tc.group, g->tc.n_group, g->tc.big, g->tc.n_big,
                 g->tc.t, g->tc.next};
  if (g->tc.n_group) {
    tc_group_kernel<<<(int)std::min<uint32_t>(g->tc.n_group, g->tc.group_grid), kTcThreads, 0, g->stream>>>(a);
    g->stats.kernel_launches++;
  }
  if (g->tc.n_big) {
    tc_big_kernel<<<(int)std::min<uint32_t>(g->tc.n_big, g->tc.big_grid), kTcThreads, 0, g->stream>>>(a);
    g->stats.kernel_launches++;
  }
  LUXB_CUDA(cudaGetLastError());
  if (g->P > 1) LUXB_NCCL(nccl().AllReduce(g->tc.t, g->tc.t, g->nv, ncclUint64, ncclSum, g->comm, g->stream));
  LUXB_CUDA(cub::DeviceReduce::Sum(g->tc.sum_tmp, g->tc.sum_bytes, g->tc.t, g->tc.total, (long long)g->nv, g->stream));
  g->stats.iterations++;
  g->stats.edges_processed += g->tc.m;
  LUXB_TRY(finish_timed(g));
  unsigned long long sum = 0;
  LUXB_CUDA(cudaMemcpyAsync(&sum, g->tc.total, 8, cudaMemcpyDeviceToHost, g->stream));
  LUXB_CUDA(cudaStreamSynchronize(g->stream));
  if (total_out) *total_out = sum / 3;  // every triangle is in t at each of its three vertices
  return 0;
}

// ---- k-core decomposition (kcore.cuh) ------------------------------------------------------------------------------
// luxb_init of a LUXB_KCORE handle: the undirected keys (undirected_keys, as for TC), then this rank's adjacency: the
// entries a -> b of every key {a, b} whose b is this rank's, sorted by (a, b) into a CSR over all nv sources
static int kcore_build(luxb_graph* g) {
  DevTmp tmp;
  const int grid = g->num_sms * 8;
  const uint32_t nv = g->nv, n_part = g->n_part;
  const int bits = pair_key_bits(nv);
  uint64_t *d_keys = nullptr, *d_alt = nullptr, m = 0;
  LUXB_TRY(undirected_keys(g, tmp, bits, &d_keys, &d_alt, &m));
  g->kc.m = m;
  tmp.release(d_alt);
  // this rank's entries: counted first, so that the two sort buffers hold this rank's share (2m / P on average), and
  // the keys go before the second buffer is allocated
  uint64_t *d_ent = nullptr, *d_ent_alt = nullptr;
  unsigned long long* d_cur = nullptr;
  LUXB_TRY(tmp.alloc(&d_cur, 1));
  const uint32_t row_right = n_part ? g->row_left + n_part - 1 : 0;
  unsigned long long n_ent = 0;
  for (int pass = 0; pass < 2; ++pass) {
    if (pass == 1) LUXB_TRY(tmp.alloc(&d_ent, n_ent));
    LUXB_CUDA(cudaMemsetAsync(d_cur, 0, 8, g->stream));
    if (m && n_part) kcore_emit_kernel<<<grid_for(m, 256, grid), 256, 0, g->stream>>>(d_keys, m, g->row_left, row_right, d_cur, d_ent);
    LUXB_CUDA(cudaGetLastError());
    LUXB_CUDA(cudaMemcpyAsync(&n_ent, d_cur, 8, cudaMemcpyDeviceToHost, g->stream));
    LUXB_CUDA(cudaStreamSynchronize(g->stream));
  }
  tmp.release(d_keys);
  LUXB_TRY(tmp.alloc(&d_ent_alt, n_ent));
  const uint64_t* d_sorted = d_ent;
  if (n_ent) {
    cub::DoubleBuffer<uint64_t> db(d_ent, d_ent_alt);
    LUXB_TRY(cub_call(tmp, g->stream, [&](void* t, size_t& b) {
      return cub::DeviceRadixSort::SortKeys(t, b, db, (long long)n_ent, 0, bits, g->stream);
    }));
    d_sorted = db.Current();
  }
  uint32_t* d_len = nullptr;
  LUXB_TRY(tmp.alloc(&d_len, nv));
  LUXB_CUDA(cudaMemsetAsync(d_len, 0, (size_t)nv * 4, g->stream));
  LUXB_TRY(gmalloc(g, &g->kc.deg0, n_part));
  LUXB_CUDA(cudaMemsetAsync(g->kc.deg0, 0, (size_t)n_part * 4, g->stream));
  LUXB_TRY(gmalloc(g, &g->kc.adj, n_ent));
  if (n_ent)
    kcore_lists_kernel<<<grid_for(n_ent, 256, grid), 256, 0, g->stream>>>(d_sorted, n_ent, g->row_left, g->kc.adj, d_len, g->kc.deg0);
  LUXB_CUDA(cudaGetLastError());
  LUXB_TRY(gmalloc(g, &g->kc.off, (uint64_t)nv + 1));
  LUXB_CUDA(cudaMemsetAsync(g->kc.off + nv, 0, 8, g->stream));
  widen_u32_to_u64_kernel<<<grid_for(nv, 256, grid), 256, 0, g->stream>>>(d_len, g->kc.off, nv);
  LUXB_TRY(cub_call(tmp, g->stream, [&](void* t, size_t& b) {
    return cub::DeviceScan::ExclusiveSum(t, b, g->kc.off, g->kc.off, (long long)nv + 1, g->stream);
  }));
  // the run's state: core (zeros until the first run), degrees, alive lists, pieces, F, its slot offsets, records
  LUXB_TRY(gmalloc(g, &g->kc.core, nv));
  LUXB_CUDA(cudaMemsetAsync(g->kc.core, 0, (size_t)nv * 4, g->stream));
  LUXB_TRY(gmalloc(g, &g->kc.deg, 2 * (uint64_t)n_part));
  for (int i = 0; i < 2; ++i) {
    LUXB_TRY(gmalloc(g, &g->kc.alive[i], n_part));
    LUXB_TRY(gmalloc(g, &g->kc.piece[i], n_part));
  }
  if (g->P > 1) LUXB_TRY(gmalloc(g, &g->kc.f, nv));
  LUXB_TRY(gmalloc(g, &g->kc.pre, (uint64_t)nv + 1));
  LUXB_TRY(gmalloc(g, &g->kc.rec, 1 + LUXB_MAX_PARTS));
  LUXB_TRY(gmalloc(g, &g->kc.h_rec, LUXB_MAX_PARTS, MemKind::kPinned));
  LUXB_TRY(gmalloc(g, &g->kc.bad, 1));
  LUXB_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, g->kc.scan_bytes, g->kc.pre, g->kc.pre, (long long)nv + 1, g->stream));
  LUXB_TRY(gmalloc(g, (char**)&g->kc.scan_tmp, g->kc.scan_bytes));
  int per_sm = 0, per_sm2 = 0;
  LUXB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kcore_scatter_kernel, kKcoreThreads, 0));
  LUXB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm2, kcore_tally_kernel, kKcoreThreads, 0));
  g->kc.grid = std::max(std::min(per_sm, per_sm2), 1) * g->num_sms;
  LUXB_CUDA(cudaStreamSynchronize(g->stream));
  return 0;
}

int luxb_kcore_run(luxb_graph* g, uint32_t* degeneracy_out) {
  LUXB_ARG(g != nullptr, "graph is NULL");
  if (!g->inited) { set_error("luxb_kcore_run before luxb_init"); return LUXB_ERR_STATE; }
  LUXB_ARG(g->cfg.app == LUXB_KCORE, "luxb_kcore_run needs a LUXB_KCORE handle (this one is app %d)", (int)g->cfg.app);
  LUXB_CUDA(cudaSetDevice(g->cfg.device));
  LUXB_CUDA(cudaEventRecord(g->ev_begin, g->stream));
  const uint32_t n_part = g->n_part, P = (uint32_t)g->P;
  const int grid = grid_for(std::max<uint32_t>(n_part, 1), 256, g->num_sms * 8);
  KcoreRec* rec = g->kc.rec;
  // every own vertex alive; core stays zero outside this rank's range, so that a sum completes it at the end
  LUXB_CUDA(cudaMemsetAsync(g->kc.core, 0, (size_t)g->nv * 4, g->stream));
  kcore_reset_kernel<<<grid, 256, 0, g->stream>>>(g->kc.core, g->kc.deg, g->kc.deg0, g->kc.alive[0], n_part, g->row_left, rec);
  kcore_tally_kernel<<<std::min(grid, g->kc.grid), kKcoreThreads, 0, g->stream>>>(g->kc.alive[0], n_part, g->kc.core, g->kc.deg,
                                                                                   g->row_left, g->kc.alive[1], rec);
  g->stats.kernel_launches += 2;
  LUXB_CUDA(cudaGetLastError());
  g->trace_active.clear();
  g->trace_pull.clear();
  int alive_cur = 0, piece_cur = 0;  // the first tally reads alive[0]
  uint32_t n_alive = 0, k = 0;
  uint64_t rounds = 0;
  std::vector<uint32_t> piece(P);
  for (;;) {
    // the one host synchronisation of a round: every rank's record
    if (P > 1) LUXB_NCCL(nccl().AllGather(rec, rec + 1, sizeof(KcoreRec), ncclUint8, g->comm, g->stream));
    LUXB_CUDA(cudaMemcpyAsync(g->kc.h_rec, P > 1 ? rec + 1 : rec, P * sizeof(KcoreRec), cudaMemcpyDeviceToHost, g->stream));
    LUXB_CUDA(cudaStreamSynchronize(g->stream));
    const KcoreRec* r = g->kc.h_rec;
    if (!r[g->cfg.rank].next) {  // the tally ran on this rank (kcore_tally_kernel): its compacted list is current
      alive_cur ^= 1;
      n_alive = r[g->cfg.rank].alive;
    }
    uint64_t next = 0, alive = 0;
    for (uint32_t p = 0; p < P; ++p) { next += r[p].next; alive += r[p].alive; }
    const uint32_t* own = g->kc.piece[piece_cur ^ 1];
    if (next) {  // the level goes on: the pieces the scatter appended
      for (uint32_t p = 0; p < P; ++p) piece[p] = r[p].next;
    } else {     // a new level: k = the least degree left, its first pieces the alive vertices at that degree
      if (!alive) break;
      uint32_t least = kKcoreUnset;
      for (uint32_t p = 0; p < P; ++p)
        if (r[p].alive) least = std::min(least, (uint32_t)(r[p].min_cnt >> 32));
      k = std::max(k, least);
      for (uint32_t p = 0; p < P; ++p) piece[p] = r[p].alive && (uint32_t)(r[p].min_cnt >> 32) == k ? (uint32_t)r[p].min_cnt : 0;
      if (piece[g->cfg.rank]) {
        kcore_select_kernel<<<grid_for(n_alive, 256, g->num_sms * 8), 256, 0, g->stream>>>(
            g->kc.alive[alive_cur], n_alive, g->kc.deg, g->row_left, k, g->kc.piece[piece_cur ^ 1], rec);
        g->stats.kernel_launches++;
      }
    }
    piece_cur ^= 1;
    uint64_t nf = 0;
    for (uint32_t p = 0; p < P; ++p) nf += piece[p];
    if (!nf) {  // every rank sees the same records, so every rank stops here: a round that removes nothing never ends
      set_error("luxb_kcore_run: round %llu at k = %u has an empty frontier with %llu vertices alive",
                (unsigned long long)rounds, k, (unsigned long long)alive);
      return LUXB_ERR_STATE;
    }
    const uint32_t mine = piece[g->cfg.rank];
    kcore_mark_kernel<<<grid_for(std::max<uint32_t>(mine, 1), 256, g->num_sms * 8), 256, 0, g->stream>>>(own, mine, k, g->kc.core, rec);
    g->stats.kernel_launches++;
    const uint32_t* f = own;
    if (P > 1) {  // the pieces in rank order, the same empty ones skipped on every rank
      LUXB_NCCL(nccl().GroupStart());
      uint64_t at = 0;
      for (uint32_t p = 0; p < P; ++p) {
        if (piece[p])
          LUXB_NCCL(nccl().Broadcast(p == (uint32_t)g->cfg.rank ? own : g->kc.f + at, g->kc.f + at, piece[p], ncclUint32, (int)p, g->comm, g->stream));
        at += piece[p];
      }
      LUXB_NCCL(nccl().GroupEnd());
      f = g->kc.f;
    }
    kcore_lengths_kernel<<<grid_for(nf + 1, 256, g->num_sms * 8), 256, 0, g->stream>>>(f, (uint32_t)nf, g->kc.off, g->kc.pre);
    size_t scan_bytes = 0;
    LUXB_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, scan_bytes, g->kc.pre, g->kc.pre, (long long)nf + 1, g->stream));
    LUXB_ARG(scan_bytes <= g->kc.scan_bytes, "k-core scan needs %zu bytes of temporary storage, %zu reserved", scan_bytes, g->kc.scan_bytes);
    LUXB_CUDA(cub::DeviceScan::ExclusiveSum(g->kc.scan_tmp, scan_bytes, g->kc.pre, g->kc.pre, (long long)nf + 1, g->stream));
    const KcoreScatterArgs sa{f, (uint32_t)nf, g->kc.pre, g->kc.off, g->kc.adj, g->kc.core, g->kc.deg, g->row_left, k,
                              g->kc.piece[piece_cur ^ 1], rec};
    kcore_scatter_kernel<<<g->kc.grid, kKcoreThreads, 0, g->stream>>>(sa);
    kcore_tally_kernel<<<std::min(grid_for(std::max<uint32_t>(n_alive, 1), kKcoreThreads, g->num_sms * 8), g->kc.grid), kKcoreThreads, 0,
                         g->stream>>>(g->kc.alive[alive_cur], n_alive, g->kc.core, g->kc.deg, g->row_left,
                                      g->kc.alive[alive_cur ^ 1], rec);
    g->stats.kernel_launches += 4;  // the scan counts as one
    LUXB_CUDA(cudaGetLastError());
    g->trace_active.push_back(nf);
    g->trace_pull.push_back((int32_t)k);
    ++rounds;
  }
  // every rank holds its own range; zeros elsewhere, so a sum completes core everywhere
  if (P > 1) LUXB_NCCL(nccl().AllReduce(g->kc.core, g->kc.core, g->nv, ncclUint32, ncclSum, g->comm, g->stream));
  g->stats.iterations += rounds;
  g->stats.edges_processed += 2 * g->kc.m;
  LUXB_TRY(finish_timed(g));
  if (degeneracy_out) *degeneracy_out = k;
  return 0;
}

// luxb_check of a LUXB_KCORE handle: this rank's vertices that are not a fixpoint of the h-index operator
static int kcore_check(luxb_graph* g, uint64_t* mistakes_out) {
  const int grid = g->num_sms * 8;
  LUXB_CUDA(cudaMemsetAsync(g->kc.bad, 0, 8, g->stream));
  LUXB_CUDA(cudaMemsetAsync(g->kc.deg, 0, (size_t)g->n_part * 8, g->stream));
  if (g->n_part) {
    kcore_check_count_kernel<<<grid, 256, 0, g->stream>>>(g->kc.off, g->kc.adj, g->nv, g->kc.core, g->row_left, g->n_part, g->kc.deg);
    kcore_check_kernel<<<grid_for(g->n_part, 256, grid), 256, 0, g->stream>>>(g->kc.core, g->row_left, g->n_part, g->kc.deg, g->kc.bad);
    LUXB_CUDA(cudaGetLastError());
  }
  unsigned long long bad = 0;
  LUXB_CUDA(cudaMemcpyAsync(&bad, g->kc.bad, 8, cudaMemcpyDeviceToHost, g->stream));
  LUXB_CUDA(cudaStreamSynchronize(g->stream));
  *mistakes_out = bad;
  return 0;
}

// ---- k-truss decomposition (truss.cuh) ------------------------------------------------------------------------------
// sup0 from scratch: TC's kernels with the edge sink over this rank's bins, summed over the ranks
static int truss_support(luxb_graph* g) {
  TrussState& t = g->tr;
  LUXB_CUDA(cudaMemsetAsync(t.sup0, 0, (size_t)t.m * 4, g->stream));
  LUXB_CUDA(cudaMemsetAsync(t.o.next, 0, 8, g->stream));
  const TcArgs a{t.o.off, t.o.dst, t.o.staged, t.o.stage_pre, t.o.group, t.o.n_group, t.o.big, t.o.n_big, nullptr, t.o.next};
  if (t.o.n_group) {
    truss_support_group_kernel<<<(int)std::min<uint32_t>(t.o.n_group, t.group_grid), kTcThreads, 0, g->stream>>>(a, t.sup0, t.oid);
    g->stats.kernel_launches++;
  }
  if (t.o.n_big) {
    truss_support_big_kernel<<<(int)std::min<uint32_t>(t.o.n_big, t.big_grid), kTcThreads, 0, g->stream>>>(a, t.sup0, t.oid);
    g->stats.kernel_launches++;
  }
  LUXB_CUDA(cudaGetLastError());
  if (g->P > 1 && t.m) LUXB_NCCL(nccl().AllReduce(t.sup0, t.sup0, t.m, ncclUint32, ncclSum, g->comm, g->stream));
  return 0;
}

// tv[v] = max τ over the edges at v
static int truss_vertex_values(luxb_graph* g) {
  TrussState& t = g->tr;
  LUXB_CUDA(cudaMemsetAsync(t.tv, 0, (size_t)g->nv * 4, g->stream));
  if (t.m) truss_vertex_kernel<<<grid_for(t.m, 256, g->num_sms * 8), 256, 0, g->stream>>>(t.ekey, t.m, t.truss, t.tv);
  LUXB_CUDA(cudaGetLastError());
  return 0;
}

// luxb_init of a LUXB_TRUSS handle: the undirected keys (undirected_keys) kept as the edge table, TC's oriented lists and
// bins (tc_orient_bins) with the edge id of every oriented position, the symmetric adjacency with edge ids, the support
static int truss_build(luxb_graph* g) {
  DevTmp tmp;
  TrussState& t = g->tr;
  const int grid = g->num_sms * 8;
  const uint32_t nv = g->nv;
  const int bits = pair_key_bits(nv);
  uint64_t *d_keys = nullptr, *d_alt = nullptr, m = 0;
  LUXB_TRY(undirected_keys(g, tmp, bits, &d_keys, &d_alt, &m));
  LUXB_ARG(m < (1ull << 32), "k-truss: %llu undirected edges, but edge ids are u32", (unsigned long long)m);
  t.m = m;
  LUXB_TRY(gmalloc(g, &t.ekey, m));
  if (m) LUXB_CUDA(cudaMemcpyAsync(t.ekey, d_keys, m * 8, cudaMemcpyDeviceToDevice, g->stream));
  uint64_t* d_range = nullptr;
  LUXB_TRY(tmp.alloc(&d_range, 2));
  truss_range_kernel<<<1, 32, 0, g->stream>>>(t.ekey, m, g->row_left, g->n_part, d_range);
  LUXB_CUDA(cudaGetLastError());
  uint64_t range[2] = {0, 0};
  LUXB_CUDA(cudaMemcpyAsync(range, d_range, 16, cudaMemcpyDeviceToHost, g->stream));
  LUXB_CUDA(cudaStreamSynchronize(g->stream));
  t.e_lo = (uint32_t)range[0];
  t.e_hi = (uint32_t)range[1];
  LUXB_TRY(tc_orient_bins(g, tmp, bits, d_keys, d_alt, m, t.o));  // orients and releases d_keys / d_alt
  LUXB_TRY(gmalloc(g, &t.oid, m));
  if (m) truss_orient_ids_kernel<<<grid, 256, 0, g->stream>>>(t.o.off, t.o.dst, nv, t.ekey, m, t.oid);
  LUXB_CUDA(cudaGetLastError());
  // the symmetric adjacency: both directions of every edge sorted by (src, dst), the edge id riding along
  uint64_t *d_k = nullptr, *d_k2 = nullptr;
  uint32_t *d_id = nullptr, *d_id2 = nullptr, *d_len = nullptr;
  LUXB_TRY(tmp.alloc(&d_k, 2 * m));
  LUXB_TRY(tmp.alloc(&d_k2, 2 * m));
  LUXB_TRY(tmp.alloc(&d_id, 2 * m));
  LUXB_TRY(tmp.alloc(&d_id2, 2 * m));
  LUXB_TRY(tmp.alloc(&d_len, nv));
  LUXB_CUDA(cudaMemsetAsync(d_len, 0, (size_t)nv * 4, g->stream));
  LUXB_TRY(gmalloc(g, &t.adj, 2 * m));
  if (m) {
    truss_emit_kernel<<<grid_for(m, 256, grid), 256, 0, g->stream>>>(t.ekey, m, d_k, d_id);
    LUXB_CUDA(cudaGetLastError());
    cub::DoubleBuffer<uint64_t> dk(d_k, d_k2);
    cub::DoubleBuffer<uint32_t> di(d_id, d_id2);
    LUXB_TRY(cub_call(tmp, g->stream, [&](void* p, size_t& b) {
      return cub::DeviceRadixSort::SortPairs(p, b, dk, di, (long long)(2 * m), 0, bits, g->stream);
    }));
    truss_lists_kernel<<<grid_for(2 * m, 256, grid), 256, 0, g->stream>>>(dk.Current(), di.Current(), 2 * m, t.adj, d_len);
    LUXB_CUDA(cudaGetLastError());
  }
  LUXB_TRY(gmalloc(g, &t.off, (uint64_t)nv + 1));
  LUXB_CUDA(cudaMemsetAsync(t.off + nv, 0, 8, g->stream));
  widen_u32_to_u64_kernel<<<grid_for(nv, 256, grid), 256, 0, g->stream>>>(d_len, t.off, nv);
  LUXB_TRY(cub_call(tmp, g->stream, [&](void* p, size_t& b) {
    return cub::DeviceScan::ExclusiveSum(p, b, t.off, t.off, (long long)nv + 1, g->stream);
  }));
  LUXB_CUDA(cudaStreamSynchronize(g->stream));
  for (void* q : {(void*)d_k, (void*)d_k2, (void*)d_id, (void*)d_id2, (void*)d_len}) tmp.release(q);
  // the run's state: support, τ (zeros until the first run), edge states, tv, alive lists, pieces, F, slots, records
  const uint32_t n_own = t.e_hi - t.e_lo;
  LUXB_TRY(gmalloc(g, &t.sup0, m));
  LUXB_TRY(gmalloc(g, &t.sup, m));
  LUXB_TRY(gmalloc(g, &t.truss, m));
  LUXB_CUDA(cudaMemsetAsync(t.truss, 0, (size_t)m * 4, g->stream));
  LUXB_TRY(gmalloc(g, &t.st, m));
  LUXB_TRY(gmalloc(g, &t.tv, nv));
  LUXB_CUDA(cudaMemsetAsync(t.tv, 0, (size_t)nv * 4, g->stream));
  for (int i = 0; i < 2; ++i) {
    LUXB_TRY(gmalloc(g, &t.alive[i], n_own));
    LUXB_TRY(gmalloc(g, &t.piece[i], n_own));
  }
  if (g->P > 1) LUXB_TRY(gmalloc(g, &t.f, m));
  LUXB_TRY(gmalloc(g, &t.pre, m + 1));
  LUXB_TRY(gmalloc(g, &t.rec, 1 + LUXB_MAX_PARTS));
  LUXB_TRY(gmalloc(g, &t.h_rec, LUXB_MAX_PARTS, MemKind::kPinned));
  LUXB_TRY(gmalloc(g, &t.bad, 1));
  LUXB_TRY(gmalloc(g, &t.o.next, 2));
  LUXB_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, t.scan_bytes, t.pre, t.pre, (long long)m + 1, g->stream));
  LUXB_TRY(gmalloc(g, (char**)&t.scan_tmp, t.scan_bytes));
  int per_sm = 0, per_sm2 = 0;
  LUXB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, truss_walk_kernel, kTrussThreads, 0));
  LUXB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm2, kcore_tally_kernel, kKcoreThreads, 0));
  t.grid = std::max(std::min(per_sm, per_sm2), 1) * g->num_sms;
  LUXB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, truss_support_group_kernel, kTcThreads, 0));
  t.group_grid = std::max(per_sm, 1) * g->num_sms;
  LUXB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, truss_support_big_kernel, kTcThreads, 0));
  t.big_grid = std::max(per_sm, 1) * g->num_sms;
  LUXB_TRY(truss_support(g));
  LUXB_CUDA(cudaStreamSynchronize(g->stream));
  return 0;
}

static int truss_handle(luxb_graph* g, const char* what) {
  LUXB_ARG(g != nullptr, "graph is NULL");
  if (!g->inited) { set_error("%s before luxb_init", what); return LUXB_ERR_STATE; }
  LUXB_ARG(g->cfg.app == LUXB_TRUSS, "%s needs a LUXB_TRUSS handle (this one is app %d)", what, (int)g->cfg.app);
  LUXB_CUDA(cudaSetDevice(g->cfg.device));
  return 0;
}

int luxb_truss_run(luxb_graph* g, uint32_t* kmax_out) {
  LUXB_TRY(truss_handle(g, "luxb_truss_run"));
  LUXB_CUDA(cudaEventRecord(g->ev_begin, g->stream));
  TrussState& t = g->tr;
  const uint32_t n_own = t.e_hi - t.e_lo, P = (uint32_t)g->P;
  KcoreRec* rec = t.rec;
  LUXB_TRY(truss_support(g));
  // every edge alive, τ unset on every rank (every rank marks the whole of F), this rank's supports from sup0
  LUXB_CUDA(cudaMemsetAsync(t.truss, 0xFF, (size_t)t.m * 4, g->stream));
  LUXB_CUDA(cudaMemsetAsync(t.st, kTrussAlive, t.m, g->stream));
  const int grid = grid_for(std::max<uint32_t>(n_own, 1), 256, g->num_sms * 8);
  kcore_reset_kernel<<<grid, 256, 0, g->stream>>>(t.truss, t.sup + t.e_lo, t.sup0 + t.e_lo, t.alive[0], n_own, t.e_lo, rec);
  kcore_tally_kernel<<<std::min(grid, t.grid), kKcoreThreads, 0, g->stream>>>(t.alive[0], n_own, t.truss, t.sup, 0, t.alive[1], rec);
  g->stats.kernel_launches += 2;
  LUXB_CUDA(cudaGetLastError());
  g->trace_active.clear();
  g->trace_pull.clear();
  int alive_cur = 0, piece_cur = 0;
  uint32_t n_alive = 0, l = 0;
  uint64_t rounds = 0;
  std::vector<uint32_t> piece(P);
  for (;;) {
    // the one host synchronisation of a round: every rank's record
    if (P > 1) LUXB_NCCL(nccl().AllGather(rec, rec + 1, sizeof(KcoreRec), ncclUint8, g->comm, g->stream));
    LUXB_CUDA(cudaMemcpyAsync(t.h_rec, P > 1 ? rec + 1 : rec, P * sizeof(KcoreRec), cudaMemcpyDeviceToHost, g->stream));
    LUXB_CUDA(cudaStreamSynchronize(g->stream));
    const KcoreRec* r = t.h_rec;
    for (uint32_t p = 0; p < P; ++p)
      if (r[p].flag) {  // a support would have gone below zero: the schedule's invariant is broken
        set_error("luxb_truss_run: round %llu at k = %u lowered a support of 0 on rank %u", (unsigned long long)rounds, l + 2, p);
        return LUXB_ERR_STATE;
      }
    if (!r[g->cfg.rank].next) {  // the tally ran on this rank: its compacted list is current
      alive_cur ^= 1;
      n_alive = r[g->cfg.rank].alive;
    }
    uint64_t next = 0, alive = 0;
    for (uint32_t p = 0; p < P; ++p) { next += r[p].next; alive += r[p].alive; }
    const uint32_t* own = t.piece[piece_cur ^ 1];
    if (next) {  // the level goes on: the pieces the walk appended
      for (uint32_t p = 0; p < P; ++p) piece[p] = r[p].next;
    } else {     // a new level: ℓ = the least support left, its first pieces the alive edges at that support
      if (!alive) break;
      uint32_t least = kKcoreUnset;
      for (uint32_t p = 0; p < P; ++p)
        if (r[p].alive) least = std::min(least, (uint32_t)(r[p].min_cnt >> 32));
      l = std::max(l, least);
      for (uint32_t p = 0; p < P; ++p) piece[p] = r[p].alive && (uint32_t)(r[p].min_cnt >> 32) == l ? (uint32_t)r[p].min_cnt : 0;
      if (piece[g->cfg.rank]) {
        kcore_select_kernel<<<grid_for(n_alive, 256, g->num_sms * 8), 256, 0, g->stream>>>(t.alive[alive_cur], n_alive, t.sup, 0, l,
                                                                                          t.piece[piece_cur ^ 1], rec);
        g->stats.kernel_launches++;
      }
    }
    piece_cur ^= 1;
    uint64_t nf = 0;
    for (uint32_t p = 0; p < P; ++p) nf += piece[p];
    if (!nf) {  // every rank sees the same records, so every rank stops here
      set_error("luxb_truss_run: round %llu at k = %u has an empty F with %llu edges alive", (unsigned long long)rounds, l + 2,
                (unsigned long long)alive);
      return LUXB_ERR_STATE;
    }
    const uint32_t* f = own;
    if (P > 1) {  // the pieces in rank order, the same empty ones skipped on every rank
      LUXB_NCCL(nccl().GroupStart());
      uint64_t at = 0;
      for (uint32_t p = 0; p < P; ++p) {
        if (piece[p])
          LUXB_NCCL(nccl().Broadcast(p == (uint32_t)g->cfg.rank ? own : t.f + at, t.f + at, piece[p], ncclUint32, (int)p, g->comm, g->stream));
        at += piece[p];
      }
      LUXB_NCCL(nccl().GroupEnd());
      f = t.f;
    }
    const int fgrid = grid_for(nf + 1, 256, g->num_sms * 8);
    truss_mark_kernel<<<fgrid, 256, 0, g->stream>>>(f, (uint32_t)nf, l + 2, t.st, t.truss, rec);
    truss_lengths_kernel<<<fgrid, 256, 0, g->stream>>>(f, (uint32_t)nf, t.ekey, t.off, t.pre);
    size_t scan_bytes = 0;
    LUXB_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, scan_bytes, t.pre, t.pre, (long long)nf + 1, g->stream));
    LUXB_ARG(scan_bytes <= t.scan_bytes, "k-truss scan needs %zu bytes of temporary storage, %zu reserved", scan_bytes, t.scan_bytes);
    LUXB_CUDA(cub::DeviceScan::ExclusiveSum(t.scan_tmp, scan_bytes, t.pre, t.pre, (long long)nf + 1, g->stream));
    const TrussWalkArgs wa{f, (uint32_t)nf, t.pre, t.ekey, t.off, t.adj, t.st, t.sup, t.e_lo, t.e_hi, l, t.piece[piece_cur ^ 1], rec};
    truss_walk_kernel<<<t.grid, kTrussThreads, 0, g->stream>>>(wa);
    truss_kill_kernel<<<fgrid, 256, 0, g->stream>>>(f, (uint32_t)nf, t.st);
    kcore_tally_kernel<<<std::min(grid_for(std::max<uint32_t>(n_alive, 1), kKcoreThreads, g->num_sms * 8), t.grid), kKcoreThreads, 0,
                         g->stream>>>(t.alive[alive_cur], n_alive, t.truss, t.sup, 0, t.alive[alive_cur ^ 1], rec);
    g->stats.kernel_launches += 6;  // the scan counts as one
    LUXB_CUDA(cudaGetLastError());
    g->trace_active.push_back(nf);
    g->trace_pull.push_back((int32_t)(l + 2));
    ++rounds;
  }
  LUXB_TRY(truss_vertex_values(g));
  g->stats.iterations += rounds;
  g->stats.edges_processed += t.m;
  LUXB_TRY(finish_timed(g));
  if (kmax_out) *kmax_out = rounds ? l + 2 : 0;
  return 0;
}

int luxb_truss_num_edges(const luxb_graph* g, uint64_t* m_out) {
  LUXB_ARG(g && m_out, "NULL argument");
  if (!g->inited) { set_error("luxb_truss_num_edges before luxb_init"); return LUXB_ERR_STATE; }
  LUXB_ARG(g->cfg.app == LUXB_TRUSS, "luxb_truss_num_edges needs a LUXB_TRUSS handle (this one is app %d)", (int)g->cfg.app);
  *m_out = g->tr.m;
  return 0;
}

int luxb_truss_edges(luxb_graph* g, luxb_vid* lo, luxb_vid* hi, uint32_t* support, uint32_t* truss, uint64_t m) {
  LUXB_TRY(truss_handle(g, "luxb_truss_edges"));
  const TrussState& t = g->tr;
  LUXB_ARG(m == t.m, "arrays of %llu edges, the graph has %llu", (unsigned long long)m, (unsigned long long)t.m);
  if (m && (lo || hi)) {
    std::vector<uint64_t> key(m);
    LUXB_CUDA(cudaMemcpyAsync(key.data(), t.ekey, m * 8, cudaMemcpyDeviceToHost, g->stream));
    LUXB_CUDA(cudaStreamSynchronize(g->stream));
    for (uint64_t i = 0; i < m; ++i) {
      if (lo) lo[i] = (uint32_t)(key[i] >> 32);
      if (hi) hi[i] = (uint32_t)key[i];
    }
  }
  if (m && support) LUXB_CUDA(cudaMemcpyAsync(support, t.sup0, m * 4, cudaMemcpyDeviceToHost, g->stream));
  if (m && truss) LUXB_CUDA(cudaMemcpyAsync(truss, t.truss, m * 4, cudaMemcpyDeviceToHost, g->stream));
  LUXB_CUDA(cudaStreamSynchronize(g->stream));
  return 0;
}

int luxb_truss_set_truss(luxb_graph* g, const uint32_t* truss, uint64_t m) {
  LUXB_TRY(truss_handle(g, "luxb_truss_set_truss"));
  LUXB_ARG(truss != nullptr || m == 0, "NULL argument");
  LUXB_ARG(m == g->tr.m, "array of %llu edges, the graph has %llu", (unsigned long long)m, (unsigned long long)g->tr.m);
  if (m) LUXB_CUDA(cudaMemcpyAsync(g->tr.truss, truss, m * 4, cudaMemcpyHostToDevice, g->stream));
  LUXB_TRY(truss_vertex_values(g));
  LUXB_CUDA(cudaStreamSynchronize(g->stream));
  return 0;
}

// luxb_check of a LUXB_TRUSS handle: this rank's edges that fail the truss check (truss_check_kernel)
static int truss_check(luxb_graph* g, uint64_t* mistakes_out) {
  const TrussState& t = g->tr;
  LUXB_CUDA(cudaMemsetAsync(t.bad, 0, 8, g->stream));
  if (t.e_hi > t.e_lo) {
    truss_check_kernel<<<g->num_sms * 8, 256, 0, g->stream>>>(t.ekey, t.e_lo, t.e_hi, t.off, t.adj, t.truss, t.bad);
    LUXB_CUDA(cudaGetLastError());
  }
  unsigned long long bad = 0;
  LUXB_CUDA(cudaMemcpyAsync(&bad, t.bad, 8, cudaMemcpyDeviceToHost, g->stream));
  LUXB_CUDA(cudaStreamSynchronize(g->stream));
  *mistakes_out = bad;
  return 0;
}

// the array luxb_get_values / luxb_set_values address: label replica, current values, betweenness scores, triangle
// counts, core numbers or vertex truss numbers
static void* values_ptr(luxb_graph* g) {
  if (app_of(g).entry == kBcRun) return g->bc.scores;
  if (g->cfg.app == LUXB_TC) return g->tc.t;
  if (g->cfg.app == LUXB_KCORE) return g->kc.core;
  if (g->cfg.app == LUXB_TRUSS) return g->tr.tv;
  return g->d_val[g->cur];  // labels: cur stays 0
}

// PageRank on several ranks exchanges only the packed transfer array every iteration: the natural-order replica is
// completed on demand (collective: every rank must make the same call)
static int refresh_replica(luxb_graph* g) {
  if (g->cfg.app == LUXB_PAGERANK && g->P > 1 && g->replica_stale) {
    LUXB_TRY(allgather_slices(g, g->d_val[g->cur], 4));
    g->replica_stale = false;
  }
  return 0;
}

int luxb_get_values(luxb_graph* g, void* host_out, size_t bytes) {
  LUXB_ARG(g && host_out, "NULL argument");
  if (!g->inited) { set_error("luxb_get_values before luxb_init"); return LUXB_ERR_STATE; }
  size_t need = (size_t)g->nv * app_of(g).vbytes;
  LUXB_ARG(bytes == need, "buffer is %zu bytes, vertex values need %zu", bytes, need);
  LUXB_CUDA(cudaSetDevice(g->cfg.device));
  LUXB_TRY(refresh_replica(g));
  const char* srcp = (const char*)values_ptr(g);
  LUXB_CUDA(cudaMemcpyAsync(host_out, srcp, need, cudaMemcpyDeviceToHost, g->stream));
  LUXB_CUDA(cudaStreamSynchronize(g->stream));
  return 0;
}

int luxb_get_local_values(luxb_graph* g, void* host_out, size_t bytes) {
  LUXB_ARG(g && (host_out || g->n_part == 0), "NULL argument");
  if (!g->inited) { set_error("luxb_get_local_values before luxb_init"); return LUXB_ERR_STATE; }
  const size_t vbytes = app_of(g).vbytes, need = (size_t)g->n_part * vbytes;
  LUXB_ARG(bytes == need, "buffer is %zu bytes, this rank's %u vertex values need %zu", bytes, g->n_part, need);
  LUXB_CUDA(cudaSetDevice(g->cfg.device));
  const char* base = (const char*)values_ptr(g);
  if (need) LUXB_CUDA(cudaMemcpyAsync(host_out, base + (size_t)g->row_left * vbytes, need, cudaMemcpyDeviceToHost, g->stream));
  LUXB_CUDA(cudaStreamSynchronize(g->stream));
  return 0;
}

// values of the vertices are in place in the current replica (whole array, or only this rank's slice): make them the
// state the next iteration starts from on every rank
static int values_installed(luxb_graph* g, bool whole_array) {
  if (g->cfg.app == LUXB_PAGERANK) {
    g->empties_done[g->cur] = false;  // caller data now sits where the constants of the edge-less vertices were
    LUXB_TRY(pagerank_publish(g, (float*)g->d_val[g->cur]));
    g->replica_stale = !whole_array && g->P > 1;
  } else {
    if (!whole_array && g->P > 1) LUXB_TRY(allgather_slices(g, values_ptr(g), app_of(g).vbytes));
    if (app_of(g).run == AppRun::kConvergence) LUXB_TRY(reset_label_state(g, true, g->cfg.start_vtx));
  }
  LUXB_CUDA(cudaStreamSynchronize(g->stream));
  return 0;
}

int luxb_set_values(luxb_graph* g, const void* host_in, size_t bytes) {
  LUXB_ARG(g && host_in, "NULL argument");
  if (!g->inited) { set_error("luxb_set_values before luxb_init"); return LUXB_ERR_STATE; }
  LUXB_ARG(app_of(g).settable, "luxb_set_values: %s computes its values from zero in %s", app_of(g).name, app_of(g).entry);
  size_t need = (size_t)g->nv * app_of(g).vbytes;
  LUXB_ARG(bytes == need, "buffer is %zu bytes, vertex values need %zu", bytes, need);
  LUXB_CUDA(cudaSetDevice(g->cfg.device));
  char* dstp = (char*)values_ptr(g);
  LUXB_CUDA(cudaMemcpyAsync(dstp, host_in, need, cudaMemcpyHostToDevice, g->stream));
  return values_installed(g, true);
}

int luxb_set_local_values(luxb_graph* g, const void* host_in, size_t bytes) {
  LUXB_ARG(g && (host_in || g->n_part == 0), "NULL argument");
  if (!g->inited) { set_error("luxb_set_local_values before luxb_init"); return LUXB_ERR_STATE; }
  LUXB_ARG(app_of(g).settable, "luxb_set_local_values: %s computes its values from zero in %s", app_of(g).name, app_of(g).entry);
  const size_t vbytes = app_of(g).vbytes, need = (size_t)g->n_part * vbytes;
  LUXB_ARG(bytes == need, "buffer is %zu bytes, this rank's %u vertex values need %zu", bytes, g->n_part, need);
  LUXB_CUDA(cudaSetDevice(g->cfg.device));
  char* dstp = (char*)values_ptr(g);
  if (need) LUXB_CUDA(cudaMemcpyAsync(dstp + (size_t)g->row_left * vbytes, host_in, need, cudaMemcpyHostToDevice, g->stream));
  return values_installed(g, false);
}

int luxb_check(luxb_graph* g, uint64_t* mistakes_out) {
  LUXB_ARG(g && mistakes_out, "NULL argument");
  if (!g->inited) { set_error("luxb_check before luxb_init"); return LUXB_ERR_STATE; }
  const AppInfo& app = app_of(g);
  LUXB_ARG(app.check || app.run != AppRun::kEntry, "luxb_check: %s has no check; it runs through %s", app.name, app.entry);
  LUXB_ARG(app.check,
           "the reference has no check for pagerank / col_filter (CHECK_TASK_ID is not registered in pull_model.inl:482-521)");
  LUXB_CUDA(cudaSetDevice(g->cfg.device));
  if (g->cfg.app == LUXB_KCORE) return kcore_check(g, mistakes_out);
  if (g->cfg.app == LUXB_TRUSS) return truss_check(g, mistakes_out);
  LUXB_CUDA(cudaMemsetAsync(g->d_counters + 1, 0, 8, g->stream));
  const uint32_t* lab = reinterpret_cast<const uint32_t*>(g->d_val[0]);
  int grid = grid_for(g->n_part, 256, g->num_sms * 8);
  if (g->n_part) {
    if (g->cfg.app == LUXB_CC)
      check_kernel<MaxLabelProgram><<<grid, 256, 0, g->stream>>>(g->d_row_end, g->d_src, g->n_part, g->row_left, g->nv, lab, g->d_counters + 1);
    else if (g->cfg.app == LUXB_SSSP)
      check_kernel<HopDistProgram><<<grid, 256, 0, g->stream>>>(g->d_row_end, g->d_src, g->n_part, g->row_left, g->nv, lab, g->d_counters + 1);
    else
      check_kernel<WeightedDistProgram><<<grid, 256, 0, g->stream>>>(g->d_row_end, g->d_src, g->n_part, g->row_left, lab, g->d_counters + 1,
                                                                     g->d_weight);
    LUXB_CUDA(cudaGetLastError());
  }
  unsigned long long bad = 0;
  LUXB_CUDA(cudaMemcpyAsync(&bad, g->d_counters + 1, 8, cudaMemcpyDeviceToHost, g->stream));
  LUXB_CUDA(cudaStreamSynchronize(g->stream));
  *mistakes_out = bad;
  return 0;
}

int luxb_stats(const luxb_graph* g, luxb_stats_t* out) {
  LUXB_ARG(g && out, "NULL argument");
  *out = g->stats;
  return 0;
}

int luxb_trace(const luxb_graph* g, uint64_t* active, int32_t* pull, int max_entries) {
  LUXB_ARG(g != nullptr, "graph is NULL");
  int n = (int)std::min<size_t>(g->trace_active.size(), (size_t)std::max(max_entries, 0));
  for (int i = 0; i < n; ++i) {
    if (active) active[i] = g->trace_active[i];
    if (pull) pull[i] = g->trace_pull[i];
  }
  return n;
}

int luxb_enable_kernel_timing(luxb_graph* g, int on) {
  LUXB_ARG(g != nullptr, "graph is NULL");
  g->kernel_timing = on != 0;
  return 0;
}

int luxb_get_out_degree(luxb_graph* g, luxb_vid* host_out, size_t bytes) {
  LUXB_ARG(g && host_out, "NULL argument");
  if (!g->inited || !g->d_deg) { set_error("out-degrees exist only for an initialised PageRank graph"); return LUXB_ERR_STATE; }
  LUXB_ARG(bytes == (size_t)g->nv * 4, "buffer must hold nv u32");
  LUXB_CUDA(cudaSetDevice(g->cfg.device));
  LUXB_CUDA(cudaMemcpyAsync(host_out, g->d_deg, bytes, cudaMemcpyDeviceToHost, g->stream));
  LUXB_CUDA(cudaStreamSynchronize(g->stream));
  return 0;
}

// dev tooling: raw gather rate over this partition's (possibly hot-packed) source ids, no reduction structure
__global__ void debug_gather_kernel(const uint32_t* __restrict__ idx, const float* __restrict__ nat, const float* __restrict__ hot,
                                    uint32_t hot_n, uint64_t m, float* out) {
  float acc = 0.f;
  uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
  for (uint64_t base = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; base < m; base += stride * 8) {
    uint32_t id[8];
    float v[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) { uint64_t i = base + k * stride; id[k] = i < m ? __ldg(idx + i) : hot_n; }
#pragma unroll
    for (int k = 0; k < 8; ++k) v[k] = __ldg(id[k] < hot_n ? hot + id[k] : nat + (id[k] - hot_n));
#pragma unroll
    for (int k = 0; k < 8; ++k) acc += v[k];
  }
  if (acc == 123.456f) out[0] = acc;
}

int luxb_debug_gather_ms(luxb_graph* g, int packed, float* ms_out) {
  LUXB_ARG(g && ms_out && g->inited && g->cfg.app == LUXB_PAGERANK && g->P == 1, "needs an initialised single-rank PageRank graph");
  LUXB_CUDA(cudaSetDevice(g->cfg.device));
  const bool use_hot = packed && g->hot_n;
  const uint32_t* idx = use_hot ? g->d_src_gather : g->d_src;
  const float* nat = use_hot && g->cold_z ? (const float*)g->d_hot + g->hot_n : (const float*)g->d_val[g->cur];
  const uint32_t hn = use_hot ? g->hot_n : 0;
  float best = 1e30f;
  for (int r = 0; r < 4; ++r) {
    LUXB_CUDA(cudaEventRecord(g->ev_begin, g->stream));
    debug_gather_kernel<<<g->num_sms * 4, 256, 0, g->stream>>>(idx, nat, (const float*)g->d_hot, hn, g->e_part, (float*)g->base.fix.d_head);
    LUXB_CUDA(cudaEventRecord(g->ev_end, g->stream));
    LUXB_CUDA(cudaStreamSynchronize(g->stream));
    float ms = 0.f;
    LUXB_CUDA(cudaEventElapsedTime(&ms, g->ev_begin, g->ev_end));
    if (r > 0 && ms < best) best = ms;
  }
  *ms_out = best;
  return 0;
}

int luxb_device_view_get(luxb_graph* g, luxb_device_view* out) {
  LUXB_ARG(g && out, "NULL argument");
  out->values = g->inited ? values_ptr(g) : nullptr;
  out->row_end = g->d_row_end;
  out->src = g->d_src;
  out->stream = g->stream;
  out->row_left = g->row_left;
  out->row_right = g->row_left + g->n_part - 1;
  out->local_edges = g->e_part;
  return 0;
}

int luxb_get_local_csc(luxb_graph* g, luxb_eid* row_end_abs, luxb_vid* src, int32_t* weight) {
  LUXB_ARG(g != nullptr, "graph is NULL");
  LUXB_CUDA(cudaSetDevice(g->cfg.device));
  if (row_end_abs && g->n_part) {
    LUXB_CUDA(cudaMemcpy(row_end_abs, g->d_row_end, (size_t)g->n_part * 8, cudaMemcpyDeviceToHost));
    for (uint32_t i = 0; i < g->n_part; ++i) row_end_abs[i] += g->col_left;
  }
  if (src && g->e_part) LUXB_CUDA(cudaMemcpy(src, g->d_src, g->e_part * 4, cudaMemcpyDeviceToHost));
  if (weight) {
    LUXB_ARG(g->d_weight != nullptr, "graph has no weights");
    if (g->e_part) LUXB_CUDA(cudaMemcpy(weight, g->d_weight, g->e_part * 4, cudaMemcpyDeviceToHost));
  }
  return 0;
}

void luxb_close(luxb_graph* g) {
  if (!g) return;
  pt_print(g);
  cudaSetDevice(g->cfg.device);
  if (g->stream) cudaStreamSynchronize(g->stream);
  if (g->stream2) cudaStreamSynchronize(g->stream2);
  if (g->d_hot) cudaCtxResetPersistingL2Cache();  // release the lines pinned for the hot copies
  p2p_unmap(g);
  if (g->stream2) cudaStreamSynchronize(g->stream2);
  if (g->comm) nccl().CommDestroy(g->comm);
  if (g->ev_pack) cudaEventDestroy(g->ev_pack);
  if (g->ev_cold) cudaEventDestroy(g->ev_cold);
  if (g->stream2) cudaStreamDestroy(g->stream2);
  if (g->ev_fork) cudaEventDestroy(g->ev_fork);
  if (g->ev_join) cudaEventDestroy(g->ev_join);
  if (g->stream_b) cudaStreamDestroy(g->stream_b);  // idle: it joins the compute stream at the end of every sweep
  for (size_t i = g->owned.size(); i-- > 0;) free_owned(g->owned[i]);  // newest first
  for (cudaEvent_t e : g->kt_events) cudaEventDestroy(e);
  if (g->ev_begin) cudaEventDestroy(g->ev_begin);
  if (g->ev_end) cudaEventDestroy(g->ev_end);
  if (g->stream) cudaStreamDestroy(g->stream);
  delete g;
}

}  // extern "C"
