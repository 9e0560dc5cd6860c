// bc.cuh — betweenness centrality (Brandes), the kernels behind luxb_bc_run (no reference counterpart).
// Per source s, after the hop levels lev[] of the BFS engine (label_iteration<HopDistProgram>):
//   level lists   : reached ids sorted stably by level -> order[], level_off[L + 1]
//   forward σ     : σ[v] = Σ σ[u] over in-edges (u, v) with lev[u] = lev[v] - 1, level by level (CSC slice)
//   backward δ    : δ[v] = σ[v] · Σ t[w] over out-edges (v, w) with lev[w] = lev[v] + 1, t[w] = (1 + δ[w]) / σ[w]
//                   (push CSR)
// One level-sum kernel serves both phases: a warp per level vertex sums f(neighbour) over its edge list in a fixed lane
// order and a fixed shuffle tree; a vertex with more than kBcSegment edges is cut into kBcSegment-edge segments whose
// fp64 partials are added in segment order by bc_combine_kernel.  No floating-point atomics: one rank is bitwise
// reproducible.  Results land in a level-ordered buffer (position j of the level), which is what the ranks exchange.
//
// Weighted betweenness centrality (LUXB_BC_WEIGHTED) runs the same sweeps over distance classes: D[] comes from
// label_iteration<WeightedDistProgram>, the reached ids are sorted stably by D and class k is one distinct distance.
// With every weight >= 1 a tight edge (D[u] + w == D[v], 64-bit, D[v] finite) always goes from a smaller class to a
// larger one, so ascending classes are a topological order of the shortest-path DAG.  The sums are the kernels above
// with the filter swapped (bc_class_sum_kernel / bc_class_hub_segments_kernel): the vertex's own D replaces the target
// and the edge's weight is read beside the neighbour id.  Lane order and shuffle tree are the same, so unit weights
// give the hop-level results bit for bit.
#pragma once
#include <stdint.h>
#include <cuda_runtime.h>
#include "common.cuh"
#include "programs.cuh"

namespace luxb {

constexpr uint32_t kBcSegment = 4096;  // edges per hub segment
constexpr int kBcThreads = 256;

// one vertex of the level whose edge list is cut into segments; segment 0 is summed by bc_level_sum_kernel
struct BcHub {
  uint32_t pos;    // position in the level
  uint32_t nseg;   // ceil(deg / kBcSegment)
  uint32_t base;   // its partials: partial[base .. base + nseg)
  uint32_t dist;   // distance classes: D of the vertex (hop levels: 0)
  uint64_t begin;  // first edge
  uint64_t deg;
};

struct BcCtl {
  uint32_t n_hub;  // hubs of the level being summed
  uint32_t n_seg;  // partial slots handed out
};

// kOut = false: in-edges of the CSC slice (end = relative row ends of this rank, ids local after - row_left), f = σ[u].
// kOut = true : out-edges of the push CSR (end = inclusive out-degree scan over all nv sources), f = (1 + δ[w]) / σ[w].
struct BcLevelArgs {
  const uint32_t* order;  // the level's vertex ids [n]
  uint32_t n;
  uint32_t row_left;      // in-edges: global id -> local row
  const uint64_t* end;
  const uint32_t* nbr;
  const uint32_t* lev;
  uint32_t target;        // neighbours at this level only
  const double* sigma;
  const double* delta;
  double* out;            // [n] the sum of each level vertex
  BcCtl* ctl;
  BcHub* hubs;
  double* partial;
  unsigned long long* edges;  // edges scanned
};

// weighted sums: the CSC weights (σ) or the push CSR's out_w (δ), aligned with nbr
struct BcClassArgs {
  BcLevelArgs a;
  const int32_t* weight;
};

// a tight edge from -> to: D[from] + w == D[to] without wrap-around, D[to] finite (so a path whose sum saturates to
// INF never matches, and an unreached tail never does: INF + w > every u32)
__device__ __forceinline__ bool bc_tight(uint32_t from, int32_t w, uint32_t to) {
  return to != kDistInf && (uint64_t)from + (uint32_t)w == to;
}

template <bool kOut>
__device__ __forceinline__ double bc_term(const BcLevelArgs& a, uint32_t w) {
  if constexpr (kOut) return (1.0 + a.delta[w]) / a.sigma[w];
  else return a.sigma[w];
}

// sum of f over edges [e0, e1) of one vertex, by one warp; every lane returns the same value.  kW: the edges kept are
// the tight ones at the vertex's distance dv (weights wt), else the neighbours on level a.target
template <bool kOut, bool kW>
__device__ __forceinline__ double bc_warp_sum(const BcLevelArgs& a, const int32_t* wt, uint32_t dv, uint64_t e0, uint64_t e1,
                                              int lane) {
  double s = 0.0;
  for (uint64_t e = e0 + lane; e < e1; e += 32) {
    const uint32_t w = __ldg(a.nbr + e);
    bool on;
    if constexpr (kW) {
      const uint32_t dw = __ldg(a.lev + w);
      const int32_t wgt = __ldg(wt + e);
      on = kOut ? bc_tight(dv, wgt, dw) : bc_tight(dw, wgt, dv);
    } else {
      on = __ldg(a.lev + w) == a.target;
    }
    if (on) s += bc_term<kOut>(a, w);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xFFFFFFFFu, s, o);  // a + b == b + a: the same sum on every lane
  return s;
}

template <bool kOut>
__device__ __forceinline__ void bc_edge_range(const BcLevelArgs& a, uint32_t v, uint64_t& e0, uint64_t& e1) {
  const uint32_t r = kOut ? v : v - a.row_left;
  e0 = r ? a.end[r - 1] : 0;
  e1 = a.end[r];
}

template <bool kOut, bool kW>
__device__ __forceinline__ void bc_level_sum(const BcLevelArgs& a, const int32_t* wt) {
  const int lane = threadIdx.x & 31;
  const uint32_t warps = gridDim.x * (kBcThreads / 32);
  unsigned long long scanned = 0;
  for (uint32_t j = blockIdx.x * (kBcThreads / 32) + threadIdx.x / 32; j < a.n; j += warps) {
    uint64_t e0, e1;
    const uint32_t v = a.order[j];
    bc_edge_range<kOut>(a, v, e0, e1);
    const uint32_t dv = kW ? __ldg(a.lev + v) : 0u;
    const uint64_t deg = e1 - e0;
    scanned += deg;
    if (deg <= kBcSegment) {
      const double s = bc_warp_sum<kOut, kW>(a, wt, dv, e0, e1, lane);
      if (lane == 0) a.out[j] = s;
      continue;
    }
    const uint32_t nseg = (uint32_t)((deg + kBcSegment - 1) / kBcSegment);
    uint32_t base = 0;
    if (lane == 0) {
      const uint32_t k = atomicAdd(&a.ctl->n_hub, 1u);
      base = atomicAdd(&a.ctl->n_seg, nseg);
      a.hubs[k] = BcHub{j, nseg, base, dv, e0, deg};
    }
    base = __shfl_sync(0xFFFFFFFFu, base, 0);
    const double s = bc_warp_sum<kOut, kW>(a, wt, dv, e0, e0 + kBcSegment, lane);
    if (lane == 0) a.partial[base] = s;
  }
  if (lane == 0 && scanned) atomicAdd(a.edges, scanned);
}

template <bool kOut>
__global__ void __launch_bounds__(kBcThreads) bc_level_sum_kernel(const __grid_constant__ BcLevelArgs a) {
  bc_level_sum<kOut, false>(a, nullptr);
}

template <bool kOut>
__global__ void __launch_bounds__(kBcThreads) bc_class_sum_kernel(const __grid_constant__ BcClassArgs c) {
  bc_level_sum<kOut, true>(c.a, c.weight);
}

// segments 1 .. nseg-1 of every hub of the level, spread over all warps of the grid
template <bool kOut, bool kW>
__device__ __forceinline__ void bc_hub_segments(const BcLevelArgs& a, const int32_t* wt) {
  const int lane = threadIdx.x & 31;
  const uint32_t W = gridDim.x * (kBcThreads / 32);
  const uint32_t gw = blockIdx.x * (kBcThreads / 32) + threadIdx.x / 32;
  const uint32_t n_hub = a.ctl->n_hub;
  uint32_t acc = 0;  // segments (past the first) of the hubs before this one
  for (uint32_t h = 0; h < n_hub; ++h) {
    const BcHub hub = a.hubs[h];
    const uint32_t extra = hub.nseg - 1;
    for (uint32_t k = (gw + W - acc % W) % W; k < extra; k += W) {
      const uint32_t s = k + 1;
      const uint64_t e0 = hub.begin + (uint64_t)s * kBcSegment;
      const uint64_t e1 = min(e0 + kBcSegment, hub.begin + hub.deg);
      const double sum = bc_warp_sum<kOut, kW>(a, wt, hub.dist, e0, e1, lane);
      if (lane == 0) a.partial[hub.base + s] = sum;
    }
    acc += extra;
  }
}

template <bool kOut>
__global__ void __launch_bounds__(kBcThreads) bc_hub_segments_kernel(const __grid_constant__ BcLevelArgs a) {
  bc_hub_segments<kOut, false>(a, nullptr);
}

template <bool kOut>
__global__ void __launch_bounds__(kBcThreads) bc_class_hub_segments_kernel(const __grid_constant__ BcClassArgs c) {
  bc_hub_segments<kOut, true>(c.a, c.weight);
}

// each hub's partials in segment order
__global__ void bc_combine_kernel(const BcCtl* __restrict__ ctl, const BcHub* __restrict__ hubs, const double* __restrict__ partial,
                                  double* __restrict__ out) {
  const uint32_t n_hub = ctl->n_hub;
  for (uint32_t h = blockIdx.x * blockDim.x + threadIdx.x; h < n_hub; h += gridDim.x * blockDim.x) {
    const BcHub hub = hubs[h];
    double s = 0.0;
    for (uint32_t k = 0; k < hub.nseg; ++k) s += partial[hub.base + k];
    out[hub.pos] = s;
  }
}

// ---- level lists ---------------------------------------------------------------------------------------------------
// deepest level reached (lev < nv)
__global__ void bc_max_level_kernel(const uint32_t* __restrict__ lev, uint32_t nv, uint32_t* __restrict__ out) {
  uint32_t m = 0;
  for (uint32_t v = blockIdx.x * blockDim.x + threadIdx.x; v < nv; v += gridDim.x * blockDim.x) {
    const uint32_t l = lev[v];
    if (l < nv && l > m) m = l;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) m = max(m, __shfl_xor_sync(0xFFFFFFFFu, m, o));
  if ((threadIdx.x & 31) == 0 && m) atomicMax(out, m);
}

// sort keys (level, or L for unreached) and ids
__global__ void bc_keys_kernel(const uint32_t* __restrict__ lev, uint32_t nv, uint32_t L, uint32_t* __restrict__ key,
                               uint32_t* __restrict__ id) {
  for (uint32_t v = blockIdx.x * blockDim.x + threadIdx.x; v < nv; v += gridDim.x * blockDim.x) {
    const uint32_t l = lev[v];
    key[v] = l < nv ? l : L;
    id[v] = v;
  }
}

// level_off[k] = first position of key k in the sorted keys (every level 0 .. L-1 is non-empty); level_off[L] = the
// number of reached vertices (preset to nv by the caller)
__global__ void bc_level_off_kernel(const uint32_t* __restrict__ key, uint32_t nv, uint32_t* __restrict__ level_off) {
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < nv; i += gridDim.x * blockDim.x)
    if (i == 0 || key[i - 1] != key[i]) level_off[key[i]] = i;
}

// ---- distance classes (weighted) ------------------------------------------------------------------------------------
// out[0] = largest finite distance, out[1] = number of reached vertices (D != INF: a distance may exceed nv)
__global__ void bc_dist_max_kernel(const uint32_t* __restrict__ dist, uint32_t nv, uint32_t* __restrict__ out) {
  uint32_t m = 0, c = 0;
  for (uint32_t v = blockIdx.x * blockDim.x + threadIdx.x; v < nv; v += gridDim.x * blockDim.x) {
    const uint32_t d = dist[v];
    if (d != kDistInf) { m = max(m, d); ++c; }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    m = max(m, __shfl_xor_sync(0xFFFFFFFFu, m, o));
    c += __shfl_xor_sync(0xFFFFFFFFu, c, o);
  }
  if ((threadIdx.x & 31) == 0 && c) {
    atomicMax(out, m);
    atomicAdd(out + 1, c);
  }
}

// sort keys (distance, or K = largest distance + 1 for unreached) and ids
__global__ void bc_dist_keys_kernel(const uint32_t* __restrict__ dist, uint32_t nv, uint32_t K, uint32_t* __restrict__ key,
                                    uint32_t* __restrict__ id) {
  for (uint32_t v = blockIdx.x * blockDim.x + threadIdx.x; v < nv; v += gridDim.x * blockDim.x) {
    const uint32_t d = dist[v];
    key[v] = d != kDistInf ? d : K;
    id[v] = v;
  }
}

// position i of the sorted keys starts a class (cub::DeviceSelect::If over the positions gives class_off)
struct BcClassHead {
  const uint32_t* key;
  __device__ __forceinline__ bool operator()(uint32_t i) const { return i == 0 || key[i - 1] != key[i]; }
};

// class_off[k] = reached for k in [classes, n): entry `classes` closes the last class, and the entries past it (the host
// reads a bound on the class count, not the count) are empty classes
__global__ void bc_class_tail_kernel(const uint32_t* __restrict__ classes, uint32_t n, uint32_t reached,
                                     uint32_t* __restrict__ class_off) {
  for (uint32_t k = *classes + blockIdx.x * blockDim.x + threadIdx.x; k < n; k += gridDim.x * blockDim.x) class_off[k] = reached;
}

struct BcSplitArgs {
  uint32_t rl[LUXB_MAX_PARTS + 1];  // first id of every partition, then nv
  int P;
};

// split[d * (P + 1) + p] = first position of level d holding an id >= rl[p] (p = P: the level's end): the ids of one
// level are ascending, so every partition owns a contiguous piece of it
__global__ void bc_split_kernel(const uint32_t* __restrict__ order, const uint32_t* __restrict__ level_off, uint32_t L,
                                const __grid_constant__ BcSplitArgs a, uint32_t* __restrict__ split) {
  const uint32_t n = L * (uint32_t)(a.P + 1);
  for (uint32_t t = blockIdx.x * blockDim.x + threadIdx.x; t < n; t += gridDim.x * blockDim.x) {
    const uint32_t d = t / (a.P + 1), p = t % (a.P + 1);
    uint32_t lo = level_off[d], hi = level_off[d + 1];
    const uint32_t bound = a.rl[p];
    while (lo < hi) {
      const uint32_t mid = lo + (hi - lo) / 2;
      if (order[mid] < bound) lo = mid + 1; else hi = mid;
    }
    split[t] = lo;
  }
}

// ---- per-level finishing --------------------------------------------------------------------------------------------
// σ of the level's vertices from their sums
__global__ void bc_sigma_finish_kernel(const uint32_t* __restrict__ order, uint32_t n, const double* __restrict__ sum,
                                       double* __restrict__ sigma) {
  for (uint32_t j = blockIdx.x * blockDim.x + threadIdx.x; j < n; j += gridDim.x * blockDim.x) sigma[order[j]] = sum[j];
}

// δ = σ · Σ t
__global__ void bc_delta_finish_kernel(const uint32_t* __restrict__ order, uint32_t n, const double* __restrict__ sum,
                                       const double* __restrict__ sigma, double* __restrict__ delta) {
  for (uint32_t j = blockIdx.x * blockDim.x + threadIdx.x; j < n; j += gridDim.x * blockDim.x) {
    const uint32_t v = order[j];
    delta[v] = sigma[v] * sum[j];
  }
}

__global__ void bc_source_kernel(double* __restrict__ sigma, uint32_t s) { sigma[s] = 1.0; }

// scores += δ over the reached vertices past the source (order[0] = s, the only level-0 vertex)
__global__ void bc_accumulate_kernel(const uint32_t* __restrict__ order, uint32_t reached, const double* __restrict__ delta,
                                     double* __restrict__ scores) {
  for (uint32_t i = 1 + blockIdx.x * blockDim.x + threadIdx.x; i < reached; i += gridDim.x * blockDim.x) {
    const uint32_t v = order[i];
    scores[v] += delta[v];
  }
}

}  // namespace luxb
