// build.cuh — one-time graph construction on the device: synthetic generators, partitioning, per-partition
// layout (relative row_end with sentinels, padded source ids), out-degrees, CSR-by-source for the push model.
// Replaces the CPU load/scan tasks and the init kernels of the reference:
//   pull_scan_task_impl  pull_model.inl:322-345      -> hist_src_kernel
//   init_push_kernel / init_push_row_ptrs / init_push_col_idxs components_gpu.cu:550-607 -> build_push_csr()
//   Graph::Graph partitioner pull_model.inl:108-131  -> partition_kernel (bit-identical bounds); balanced_cut_kernel
//                                                      for the optional cost-balanced work split
// plus the hot-packed gather layout, and the kernels of PageRank's packed exchange (pack_push / chunk_pull / hot_permute:
// those three run every iteration).  The rest is not on the timed hot path; device-wide scans/sorts use CUB (bundled with CUDA, as the reference itself does).
#pragma once
#include "common.cuh"

namespace luxb {

// ---- deterministic counter-based generators; MUST match oracle/lux_oracle.c lo_rmat_edge bit for bit ---------
#define LUXB_RMAT_T0 37356u
#define LUXB_RMAT_T1 49807u
#define LUXB_RMAT_T2 62259u

__device__ __forceinline__ void rmat_edge(uint64_t seed_mixed, uint64_t i, int scale, uint32_t nv, uint32_t& src,
                                          uint32_t& dst) {
  uint64_t h0 = splitmix64(seed_mixed ^ i);
  for (uint64_t attempt = 0;; ++attempt) {
    uint64_t ha = splitmix64(h0 + attempt);
    uint32_t s = 0, d = 0;
    uint64_t w = 0;
    for (int lvl = 0; lvl < scale; ++lvl) {
      if ((lvl & 3) == 0) w = splitmix64(ha ^ ((uint64_t)(lvl / 4 + 1) * 0xA0761D6478BD642Full));
      uint32_t r = (uint32_t)(w & 0xFFFFu);
      w >>= 16;
      uint32_t sb = r >= LUXB_RMAT_T1 ? 1u : 0u;
      uint32_t db = (r >= LUXB_RMAT_T0 && r < LUXB_RMAT_T1) || r >= LUXB_RMAT_T2 ? 1u : 0u;
      s = (s << 1) | sb;
      d = (d << 1) | db;
    }
    if (s < nv && d < nv) { src = s; dst = d; return; }
  }
}

__device__ __forceinline__ int32_t edge_weight(uint64_t seed, uint32_t src, uint32_t dst) {
  uint64_t h = splitmix64(splitmix64(seed ^ 0x5bd1e995u) ^ (((uint64_t)dst << 32) | src));
  return (int32_t)(1 + (h >> 33) % 5);
}

// weighted SSSP on RMAT: a directed weight in [1, 255] that depends only on (seed, src, dst); MUST match
// tests/weighted_oracle.c wo_rmat_weight bit for bit
__device__ __forceinline__ int32_t rmat_weight(uint64_t seed, uint32_t src, uint32_t dst) {
  uint64_t h = splitmix64(splitmix64(seed ^ 0x9E3779B97F4A7C15ull) ^ (((uint64_t)dst << 32) | src));
  return (int32_t)(1 + (h >> 32) % 255);
}

__device__ __forceinline__ void bipartite_edge(uint64_t seed_mixed, uint64_t j, uint32_t users, uint32_t items,
                                               uint32_t& user, uint32_t& item) {
  uint64_t h1 = splitmix64(seed_mixed ^ j);
  uint64_t h2 = splitmix64(h1 ^ 0xA0761D6478BD642Full);
  user = (uint32_t)(((h1 >> 32) * (uint64_t)users) >> 32);
  uint64_t a = h2 & 0xFFFFFFFFull, b = h2 >> 32;
  uint64_t m = (a * b) >> 32;
  item = users + (uint32_t)((m * (uint64_t)items) >> 32);
}

// kind 0: RMAT (ne edges).  kind 1: bipartite (ne = 2*ratings; edge 2j = user->item, 2j+1 = item->user).
struct GenSpec {
  int kind;
  int scale;
  uint32_t nv;
  uint64_t ne;
  uint64_t seed;
  uint32_t users, items;
};

__device__ __forceinline__ void gen_edge(const GenSpec& g, uint64_t seed_mixed, uint64_t e, uint32_t& s, uint32_t& d) {
  if (g.kind == 0) {
    rmat_edge(seed_mixed, e, g.scale, g.nv, s, d);
  } else {
    uint32_t u, it;
    bipartite_edge(seed_mixed, e >> 1, g.users, g.items, u, it);
    if (e & 1) { s = it; d = u; } else { s = u; d = it; }
  }
}

__global__ void gen_count_indeg_kernel(GenSpec g, uint32_t* __restrict__ indeg) {
  uint64_t seed_mixed = splitmix64(g.seed);
  for (uint64_t e = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; e < g.ne; e += (uint64_t)gridDim.x * blockDim.x) {
    uint32_t s, d;
    gen_edge(g, seed_mixed, e, s, d);
    atomicAdd(indeg + d, 1u);
  }
}

// emit key = (dst - row_left) << 32 | src for the edges whose destination lies in [row_left, row_left + n_part)
__global__ void gen_emit_keys_kernel(GenSpec g, uint32_t row_left, uint32_t n_part, unsigned long long* cursor,
                                     uint64_t* __restrict__ keys, uint64_t capacity) {
  uint64_t seed_mixed = splitmix64(g.seed);
  const unsigned lane = threadIdx.x & 31;
  uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
  uint64_t rounds = (g.ne + stride - 1) / stride;
  for (uint64_t r = 0; r < rounds; ++r) {
    uint64_t e = r * stride + (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    bool mine = false;
    uint64_t key = 0;
    if (e < g.ne) {
      uint32_t s, d;
      gen_edge(g, seed_mixed, e, s, d);
      if (d >= row_left && d - row_left < n_part) { mine = true; key = ((uint64_t)(d - row_left) << 32) | s; }
    }
    unsigned m = __ballot_sync(0xffffffffu, mine);  // warp-aggregated append
    if (m) {
      unsigned long long base = 0;
      int leader = __ffs(m) - 1;
      if ((int)lane == leader) base = atomicAdd(cursor, (unsigned long long)__popc(m));
      base = __shfl_sync(0xffffffffu, base, leader);
      if (mine) {
        uint64_t pos = base + __popc(m & ((1u << lane) - 1));
        if (pos < capacity) keys[pos] = key;
      }
    }
  }
}

__global__ void keys_to_src_kernel(const uint64_t* __restrict__ keys, uint64_t n, uint32_t* __restrict__ src,
                                   int32_t* __restrict__ weight, uint64_t seed, uint32_t row_left) {
  for (uint64_t e = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; e < n; e += (uint64_t)gridDim.x * blockDim.x) {
    uint64_t k = keys[e];
    uint32_t s = (uint32_t)k;
    src[e] = s;
    if (weight) {
      uint32_t d = (uint32_t)(k >> 32) + row_left;
      uint32_t lo = s < d ? s : d, hi = s < d ? d : s;
      weight[e] = edge_weight(seed, lo, hi);
    }
  }
}

// RMAT weights of the sorted keys ((dst - row_left) << 32 | src), in CSC order
__global__ void keys_to_rmat_weight_kernel(const uint64_t* __restrict__ keys, uint64_t n, int32_t* __restrict__ weight, uint64_t seed,
                                           uint32_t row_left) {
  for (uint64_t e = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; e < n; e += (uint64_t)gridDim.x * blockDim.x) {
    uint64_t k = keys[e];
    weight[e] = rmat_weight(seed, (uint32_t)k, (uint32_t)(k >> 32) + row_left);
  }
}

// The reference's greedy edge-balanced split (pull_model.inl:108-131): walking v upward, close a partition AT v
// (inclusive) as soon as the edges accumulated since `left` exceed cap = ceil(ne/P).  Since the running count is
// row_end[v] - base, each cut is the smallest v with row_end[v] - base > cap: a binary search.  Trailing remainder
// becomes the last partition; if fewer than P result, the rest are empty (row_left = nv, n = 0).
__global__ void partition_kernel(const uint64_t* __restrict__ row_end, uint32_t nv, uint64_t ne, int P,
                                 uint32_t* row_left, uint32_t* n_part, uint64_t* col_left, int* count_out) {
  if (blockIdx.x != 0 || threadIdx.x != 0) return;
  uint64_t cap = (ne + P - 1) / P;
  uint32_t left = 0;
  int count = 0, found_adjust = 0;
  while (left < nv && count < P) {
    uint64_t base = left == 0 ? 0 : row_end[left - 1];
    uint32_t lo = left, hi = nv;  // first v in [left, nv) with row_end[v] - base > cap, or nv
    while (lo < hi) {
      uint32_t mid = lo + (hi - lo) / 2;
      if (row_end[mid] - base > cap) hi = mid; else lo = mid + 1;
    }
    if (lo < nv) {
      row_left[count] = left; n_part[count] = lo - left + 1; col_left[count] = base; ++count;
      left = lo + 1;
    } else {
      // remainder: always kept (see host_partition in api.cu); only counted as "found" when it holds edges
      if (row_end[nv - 1] - base == 0) --found_adjust;
      row_left[count] = left; n_part[count] = nv - left; col_left[count] = base; ++count;
      left = nv;
    }
  }
  *count_out = count + found_adjust;
  for (int p = count; p < P; ++p) { row_left[p] = nv; n_part[p] = 0; col_left[p] = ne; }
}

// cost-balanced work split (api.cu: vertex_cost): per-vertex cost, and the cut points on its inclusive prefix
__global__ void vertex_cost_kernel(const uint64_t* __restrict__ row_end, uint32_t nv, uint32_t hub_indeg, uint64_t* __restrict__ cost) {
  for (uint64_t v = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; v < nv; v += (uint64_t)gridDim.x * blockDim.x) {
    const uint64_t d = row_end[v] - (v ? row_end[v - 1] : 0);
    cost[v] = 8 + (d >= hub_indeg ? 4 : 7) * d;
  }
}
__global__ void balanced_cut_kernel(const uint64_t* __restrict__ cost_prefix, const uint64_t* __restrict__ row_end, uint32_t nv, uint64_t ne,
                                    int P, uint32_t* row_left, uint32_t* n_part, uint64_t* col_left) {
  if (blockIdx.x || threadIdx.x) return;
  const uint64_t total = cost_prefix[nv - 1];
  uint32_t left = 0;
  int p = 0;
  for (; p < P - 1 && left < nv; ++p) {
    // smallest v >= left with prefix[v] * P >= total * (p + 1)  (same rule as host_balanced_partition)
    uint32_t lo = left, hi = nv - 1;
    while (lo < hi) {
      const uint32_t mid = lo + (hi - lo) / 2;
      if (cost_prefix[mid] * (uint64_t)P >= total * (uint64_t)(p + 1)) hi = mid; else lo = mid + 1;
    }
    row_left[p] = left; n_part[p] = lo - left + 1; col_left[p] = left ? row_end[left - 1] : 0;
    left = lo + 1;
  }
  if (left < nv || p == P - 1) {
    row_left[p] = left < nv ? left : nv; n_part[p] = left < nv ? nv - left : 0;
    col_left[p] = left < nv ? (left ? row_end[left - 1] : 0) : ne;
    ++p;
  }
  for (; p < P; ++p) { row_left[p] = nv; n_part[p] = 0; col_left[p] = ne; }
}

__global__ void widen_u32_to_u64_kernel(const uint32_t* __restrict__ in, uint64_t* __restrict__ out, uint64_t n) {
  for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) out[i] = in[i];
}

__global__ void narrow_u64_to_u32_kernel(const uint64_t* __restrict__ in, uint64_t n_in, uint32_t* __restrict__ out, uint64_t n_out) {
  for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n_out; i += (uint64_t)gridDim.x * blockDim.x)
    out[i] = i < n_in ? (uint32_t)in[i] : 0xFFFFFFFFu;
}

// local layout: rel[i] = row_end_global[row_left + i] - col_left for i < n_part, then 4 sentinels (~0)
__global__ void rowend_rel_kernel(const uint64_t* __restrict__ row_end_global, uint32_t row_left, uint32_t n_part,
                                  uint64_t col_left, uint64_t* __restrict__ rel) {
  for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < (uint64_t)n_part + 4;
       i += (uint64_t)gridDim.x * blockDim.x)
    rel[i] = i < n_part ? row_end_global[row_left + i] - col_left : ~0ull;
}

// input validation on the device: number of source ids >= nv in this rank's slice
__global__ void src_out_of_range_kernel(const uint32_t* __restrict__ src, uint64_t n, uint32_t nv, unsigned long long* __restrict__ bad) {
  unsigned long long c = 0;
  for (uint64_t e = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; e < n; e += (uint64_t)gridDim.x * blockDim.x) c += src[e] >= nv;
  if (c) atomicAdd(bad, c);
}

// number of negative weights in this rank's slice (weighted SSSP needs w >= 0)
__global__ void negative_weight_kernel(const int32_t* __restrict__ w, uint64_t n, unsigned long long* __restrict__ bad) {
  unsigned long long c = 0;
  for (uint64_t e = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; e < n; e += (uint64_t)gridDim.x * blockDim.x) c += w[e] < 0;
  if (c) atomicAdd(bad, c);
}

// number of weights below `lo` in this rank's slice (weighted betweenness centrality needs w >= 1)
__global__ void light_weight_kernel(const int32_t* __restrict__ w, uint64_t n, int32_t lo, unsigned long long* __restrict__ bad) {
  unsigned long long c = 0;
  for (uint64_t e = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; e < n; e += (uint64_t)gridDim.x * blockDim.x) c += w[e] < lo;
  if (c) atomicAdd(bad, c);
}

__global__ void hist_src_kernel(const uint32_t* __restrict__ src, uint64_t n, uint32_t* __restrict__ cnt) {
  for (uint64_t e = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; e < n; e += (uint64_t)gridDim.x * blockDim.x)
    atomicAdd(cnt + src[e], 1u);
}

// dst (global id) of every local edge: upper_bound over the relative row_end array
__global__ void edge_dst_kernel(const uint64_t* __restrict__ row_end_rel, uint32_t n_part, uint64_t e_part,
                                uint32_t row_left, uint32_t* __restrict__ dst) {
  for (uint64_t e = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; e < e_part; e += (uint64_t)gridDim.x * blockDim.x) {
    uint32_t lo = 0, hi = n_part;  // first i with row_end_rel[i] > e
    while (lo < hi) {
      uint32_t mid = lo + (hi - lo) / 2;
      if (row_end_rel[mid] > e) hi = mid; else lo = mid + 1;
    }
    dst[e] = row_left + lo;
  }
}

template <class T>
__global__ void fill_kernel(T* p, uint64_t n, T v) {
  for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) p[i] = v;
}

__global__ void iota_kernel(uint32_t* p, uint64_t n) {
  for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) p[i] = (uint32_t)i;
}

// ---- hot-packed gather array (PageRank) -------------------------------------------------------------------------
// Random 4-byte gathers are bounded by the DRAM random-access rate unless they hit
// L2.  Vertices are gathered in proportion to their out-degree, so the H vertices with the largest
// out-degree are given a second, CONTIGUOUS home at the front of the value array Z = [hot copy (H) | natural (nv)]
// and every source id is rewritten to point there: src' = rank(v) if hot else H + v.  Hot sectors then hold 8 hot
// values instead of 1, the hot working set fits L2 (and the TLB reach), and cold gathers keep their natural order.
__global__ void degree_hist_kernel(const uint32_t* __restrict__ deg, uint32_t nv, uint32_t cap, unsigned long long* __restrict__ hist) {
  for (uint64_t v = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; v < nv; v += (uint64_t)gridDim.x * blockDim.x) {
    uint32_t d = deg[v];
    atomicAdd(hist + (d < cap ? d : cap), 1ull);
  }
}

struct PartTable {
  uint32_t rl[LUXB_MAX_PARTS];
  uint32_t np[LUXB_MAX_PARTS];
  int P;
};
__device__ __forceinline__ int owner_of(const PartTable& pt, uint32_t v) {
  int o = 0;
  for (int p = 0; p < pt.P; ++p)
    if (pt.np[p] && v >= pt.rl[p]) o = p;
  return o;
}

// keys/ids of the hot vertices only (compacted with a warp-aggregated cursor).  key = inverted out-degree: ascending
// (key, id) = GLOBAL hotness order (the source-blocked sweep cuts it into blocks, panel.cuh); per_owner counts how many
// hot vertices each partition owns (the packed exchange ships them grouped by owner, see owner_keys_kernel).
__global__ void hot_select_kernel(const uint32_t* __restrict__ deg, uint32_t nv, uint32_t tau, PartTable pt, unsigned int* cursor,
                                  unsigned int* __restrict__ per_owner, uint64_t* __restrict__ keys, uint32_t* __restrict__ ids,
                                  uint32_t capacity) {
  const unsigned lane = threadIdx.x & 31;
  uint64_t n_round = ((uint64_t)nv + 31) & ~31ull;
  for (uint64_t v = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; v < n_round; v += (uint64_t)gridDim.x * blockDim.x) {
    bool hot = v < nv && deg[v] >= tau;
    unsigned m = __ballot_sync(0xffffffffu, hot);
    if (m) {
      unsigned base = 0;
      if (lane == 0) base = atomicAdd(cursor, (unsigned)__popc(m));
      base = __shfl_sync(0xffffffffu, base, 0);
      if (hot) {
        unsigned pos = base + __popc(m & ((1u << lane) - 1));
        int o = owner_of(pt, (uint32_t)v);
        atomicAdd(per_owner + o, 1u);
        if (pos < capacity) { keys[pos] = 0xFFFFFFFFu - deg[v]; ids[pos] = (uint32_t)v; }
      }
    }
  }
}

__global__ void gather_map_init_kernel(uint32_t* __restrict__ map, uint32_t nv, uint32_t H) {
  for (uint64_t v = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; v < nv; v += (uint64_t)gridDim.x * blockDim.x) map[v] = H + (uint32_t)v;
}
__global__ void gather_map_hot_kernel(uint32_t* __restrict__ map, const uint32_t* __restrict__ order, uint32_t H) {
  for (uint64_t h = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; h < H; h += (uint64_t)gridDim.x * blockDim.x) map[order[h]] = (uint32_t)h;
}
__global__ void remap_src_kernel(const uint32_t* __restrict__ src, uint64_t n, const uint32_t* __restrict__ map, uint32_t* __restrict__ out) {
  for (uint64_t e = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; e < n; e += (uint64_t)gridDim.x * blockDim.x) out[e] = map[src[e]];
}
// refresh hot copies [h0, h1) from the natural-order values: hot[h] = nat[order[h]]
template <class T>
__global__ void hot_refresh_kernel(T* __restrict__ hot, const T* __restrict__ nat, const uint32_t* __restrict__ order, uint32_t h0,
                                   uint32_t h1) {
  for (uint64_t h = (uint64_t)h0 + (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; h < h1; h += (uint64_t)gridDim.x * blockDim.x)
    hot[h] = nat[order[h]];
}

// ---- packed exchange (PageRank, nranks > 1) -------------------------------------------------------------------------
// Only vertices that are ever gathered (out-degree > 0) are exchanged, in a packed transfer array
//   XT = [ hot values grouped by owner (H) | cold-active values (0 < deg < tau) in natural id order = grouped by owner ]
// so that every owner's share is two contiguous ranges.  Cold gathers index XT's cold part directly; the hot part is
// permuted into the globally hotness-ordered copy the kernels gather from (zperm).  Reference precedent: only the
// in-neighbours of a partition are refreshed (in_vtxs / load_kernel, pagerank_gpu.cu:229-242, :34-47).
__global__ void cold_flag_kernel(const uint32_t* __restrict__ deg, uint32_t nv, uint32_t tau, uint32_t* __restrict__ flag) {
  for (uint64_t v = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; v < nv; v += (uint64_t)gridDim.x * blockDim.x)
    flag[v] = (deg[v] > 0 && deg[v] < tau) ? 1u : 0u;
}
__global__ void gather_map_compact_kernel(uint32_t* __restrict__ map, const uint32_t* __restrict__ coldrank, uint32_t nv, uint32_t H) {
  for (uint64_t v = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; v < nv; v += (uint64_t)gridDim.x * blockDim.x) map[v] = H + coldrank[v];
}
__global__ void owner_keys_kernel(const uint32_t* __restrict__ hot_order, uint32_t H, PartTable pt, uint32_t* __restrict__ keys,
                                  uint32_t* __restrict__ ranks) {
  for (uint64_t r = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; r < H; r += (uint64_t)gridDim.x * blockDim.x) {
    keys[r] = (uint32_t)owner_of(pt, hot_order[r]);
    ranks[r] = (uint32_t)r;
  }
}
// pack list of this rank: local indices of [its hot vertices in transfer order | its cold-active vertices ascending]
__global__ void pack_list_hot_kernel(const uint32_t* __restrict__ hot_order, const uint32_t* __restrict__ zperm, uint32_t h0, uint32_t n,
                                     uint32_t row_left, uint32_t* __restrict__ list) {
  for (uint64_t k = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; k < n; k += (uint64_t)gridDim.x * blockDim.x)
    list[k] = hot_order[zperm[h0 + k]] - row_left;
}
__global__ void pack_list_cold_kernel(const uint32_t* __restrict__ flag, const uint32_t* __restrict__ coldrank, uint32_t row_left,
                                      uint32_t n_part, uint32_t c0, uint32_t* __restrict__ list) {
  for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n_part; i += (uint64_t)gridDim.x * blockDim.x)
    if (flag[row_left + i]) list[coldrank[row_left + i] - c0] = (uint32_t)i;
}
// per iteration: dst[k] = x_local[list[k]]
template <class T>
__global__ void pack_values_kernel(const T* __restrict__ x_local, const uint32_t* __restrict__ list, uint32_t n_hot, uint32_t n_cold,
                                   T* __restrict__ dst_hot, T* __restrict__ dst_cold) {
  const uint64_t n = (uint64_t)n_hot + n_cold;
  for (uint64_t k = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; k < n; k += (uint64_t)gridDim.x * blockDim.x) {
    const T v = x_local[list[k]];
    if (k < n_hot) dst_hot[k] = v; else dst_cold[k - n_hot] = v;
  }
}
// step 1 of the balanced all-gather fused into the pack: every owned entry is stored straight into the transfer array of the
// rank that HOLDS its equal chunk (remote NVLink stores, coalesced: consecutive entries sit in consecutive positions) —
// one kernel launch instead of a local pack plus 2 (P - 1) peer cudaMemcpyAsync calls (at 8 ranks the iteration was bound
// by the HOST issuing ~45 API calls).
template <class T>
struct PackPushArgs {
  const T* x_local;        // this rank's new values, local order
  const uint32_t* list;    // local indices of [hot owned | cold-active owned] vertices in transfer order
  uint32_t n_hot, n_cold;
  uint64_t hot_pos0, cold_pos0;   // position of the first owned entry inside the hot / cold region
  uint64_t hot_chunk, cold_chunk; // equal chunk sizes (elements) of the two regions
  uint64_t cold_base;             // offset of the cold region inside XT
  T* xt[LUXB_MAX_PARTS];          // every rank's transfer array (own rank included)
  int P;
};
// kDirect: every owned entry goes to EVERY rank's transfer array (P coalesced store streams; no pull step afterwards)
template <class T, bool kDirect>
__global__ void pack_push_kernel(const __grid_constant__ PackPushArgs<T> a) {
  const uint64_t n = (uint64_t)a.n_hot + a.n_cold;
  for (uint64_t k = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; k < n; k += (uint64_t)gridDim.x * blockDim.x) {
    const T v = a.x_local[a.list[k]];
    const bool hot = k < a.n_hot;
    const uint64_t pos = hot ? a.hot_pos0 + k : a.cold_pos0 + (k - a.n_hot);
    const uint64_t at = hot ? pos : a.cold_base + pos;
    if constexpr (kDirect) {
      for (int q = 0; q < a.P; ++q) a.xt[q][at] = v;
    } else {
      a.xt[pos / (hot ? a.hot_chunk : a.cold_chunk)][at] = v;
    }
  }
}

// Barrier between the ranks of one box without a library call or a host round trip: lane k stores this barrier's epoch
// into word `me` of rank k's flag array (system-scope release, over NVLink) and spins on word k of its own array.  The
// kernels before it in the stream have completed, so their remote stores are ordered before the flag (release is
// cumulative); kernels after it see what the peers wrote before THEIR flag stores.  A peer that never arrives (its
// process died) releases the spin after timeout_ns (30 s, LUXB_BARRIER_TIMEOUT_S) with *err set — the GPU is never left
// hanging.
struct FlagBarrierArgs {
  uint32_t* peer[LUXB_MAX_PARTS];  // every rank's flag array
  uint32_t* mine;
  uint32_t* err;
  int P, me;
  uint32_t epoch;
  uint64_t timeout_ns;
};
__global__ void flag_barrier_kernel(const __grid_constant__ FlagBarrierArgs a) {
  const int k = threadIdx.x;
  if (k >= a.P || k == a.me) return;
  __threadfence_system();
  asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(a.peer[k] + a.me), "r"(a.epoch) : "memory");
  uint64_t t0, t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t0));
  for (;;) {
    uint32_t f;
    asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(f) : "l"(a.mine + k) : "memory");
    if ((int32_t)(f - a.epoch) >= 0) break;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    if (t - t0 > a.timeout_ns) { *a.err = 1u + (uint32_t)k; break; }
  }
}

// hot part of the transfer array (owner-grouped) -> globally hotness-ordered copy
template <class T>
__global__ void hot_permute_kernel(T* __restrict__ hot, const T* __restrict__ xt_hot, const uint32_t* __restrict__ zperm, uint32_t H) {
  for (uint64_t k = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; k < H; k += (uint64_t)gridDim.x * blockDim.x) hot[zperm[k]] = xt_hot[k];
}

// step 2 of the balanced all-gather without a library collective: after the barrier every rank PULLS the equal chunks it
// does not hold from their holders' transfer arrays over NVLink — 128-bit peer loads from all P - 1 peers concurrently
// (64 KB slabs dealt round-robin over the peers), stores to local HBM.  Chunk k sits at offset k * chunk in every XT.
struct ChunkPullArgs {
  float* dst;                         // this rank's XT region
  const float* src[LUXB_MAX_PARTS];   // every rank's XT region (peer pointers from cudaIpcOpenMemHandle)
  uint64_t chunk;                     // elements per chunk (multiple of 32)
  int P, me;
};
__global__ void __launch_bounds__(512) chunk_pull_kernel(const __grid_constant__ ChunkPullArgs a) {
  constexpr int kDepth = 8;                  // 128-bit peer loads in flight per thread: NVLink latency, not issue, is the bound
  constexpr uint64_t kSlab = 512 * kDepth;   // float4 per slab
  const uint64_t v4 = a.chunk / 4;
  const uint64_t slabs_per_chunk = (v4 + kSlab - 1) / kSlab;
  const uint64_t units = slabs_per_chunk * (uint64_t)(a.P - 1);
  for (uint64_t u = blockIdx.x; u < units; u += gridDim.x) {
    const int q = (int)(u % (uint64_t)(a.P - 1));
    const int k = q < a.me ? q : q + 1;
    const uint64_t j0 = (u / (uint64_t)(a.P - 1)) * kSlab + threadIdx.x;
    const float4* s = reinterpret_cast<const float4*>(a.src[k] + (uint64_t)k * a.chunk);
    float4* d = reinterpret_cast<float4*>(a.dst + (uint64_t)k * a.chunk);
    float4 r[kDepth];
#pragma unroll
    for (int i = 0; i < kDepth; ++i)
      if (j0 + (uint64_t)i * 512 < v4) r[i] = s[j0 + (uint64_t)i * 512];
#pragma unroll
    for (int i = 0; i < kDepth; ++i)
      if (j0 + (uint64_t)i * 512 < v4) d[j0 + (uint64_t)i * 512] = r[i];
  }
}

// PageRank init: x0[v] = (1/nv)/deg[v], or 1/nv for deg 0  (pagerank_gpu.cu:255-259)
__global__ void pr_init_kernel(const uint32_t* __restrict__ deg, uint32_t nv, float* __restrict__ x) {
  float rank = __fdiv_rn(1.0f, (float)nv);
  for (uint64_t v = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; v < nv; v += (uint64_t)gridDim.x * blockDim.x) {
    uint32_t d = deg[v];
    x[v] = d == 0 ? rank : __fdiv_rn(rank, (float)d);
  }
}

}  // namespace luxb
