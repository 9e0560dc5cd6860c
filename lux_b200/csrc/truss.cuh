// truss.cuh — k-truss decomposition (no reference counterpart), the kernels behind luxb_truss_run.
// The graph is LUXB_TC's: the CSC's directed edges read as an undirected simple graph with m edges, edge id = rank of
// (lo, hi) among the edges in ascending order.  sup(e) is the number of triangles that contain e; τ(e) the largest
// k >= 2 such that e lies in a subgraph whose every edge is in at least k - 2 triangles of that subgraph.
//
// Construction (luxb_init, once): the distinct undirected keys (shared with TC and k-core), kept as the edge table;
// TC's oriented out-lists and bins of this rank's range (tc_orient_bins), with the edge id of every oriented position;
// and the full symmetric adjacency, one (neighbour << 32 | edge id) entry per direction of every edge, ascending
// neighbours inside each list (every rank holds all of it).
//
// Support (hot path 1): TC's grouped and big kernels with TrussEdgeSink: every count they make belongs to one oriented
// edge, and goes to sup[eid[position]] instead of t[].  Each rank counts at the oriented edges whose tail is in its
// range; a u32 sum over the ranks completes sup.
//
// The peel (hot path 2), level-synchronous, with ℓ = k - 2: ℓ = 0; while an edge is alive: ℓ = max(ℓ, min sup over the
// alive edges); repeat: F = {alive e : sup(e) <= ℓ}, stop if F is empty; τ[F] = ℓ + 2; every triangle whose three edges
// were alive at the start of the round and which has an edge in F lowers the support of each of its edges not in F by
// one, from the F edge of the smallest id only; remove F.  Per round: mark F dying (state 1) before any walk; flatten the
// triangle walks of F over the grid (for F edge {u, v}, the slots are the entries of the shorter of the two lists, each
// looked up in the longer one by binary search), skip triangles with a dead edge, apply the smallest-F-id rule and
// atomicSub the non-F edges this rank owns; an edge joins the next piece iff the old value was ℓ + 1 (exactly once,
// warp-aggregated); then mark F dead (state 2).  The alive list, its tally and the level-start select are k-core's
// (kcore.cuh) over this rank's edge ids, with τ in the role of core and sup in that of deg.
#pragma once
#include <stdint.h>
#include <cuda_runtime.h>
#include "common.cuh"
#include "kcore.cuh"
#include "tc.cuh"

namespace luxb {

constexpr int kTrussThreads = 256;
constexpr uint8_t kTrussAlive = 0, kTrussDying = 1, kTrussDead = 2;

// support sink of TC's kernels: oriented position p -> its edge
struct TrussEdgeSink {
  static constexpr bool kPerEdge = true;
  uint32_t* sup;
  const uint32_t* eid;
  __device__ __forceinline__ void add(uint64_t p, uint32_t c) const { atomicAdd(sup + eid[p], c); }
};

__global__ void __launch_bounds__(kTcThreads) truss_support_group_kernel(const __grid_constant__ TcArgs a, uint32_t* sup,
                                                                         const uint32_t* eid) {
  tc_group_body(a, TrussEdgeSink{sup, eid});
}

__global__ void __launch_bounds__(kTcThreads) truss_support_big_kernel(const __grid_constant__ TcArgs a, uint32_t* sup,
                                                                       const uint32_t* eid) {
  tc_big_body(a, TrussEdgeSink{sup, eid});
}

// first i in [b, e) with key[i] >= want
__device__ __forceinline__ uint64_t truss_lower_bound(const uint64_t* __restrict__ key, uint64_t b, uint64_t e, uint64_t want) {
  while (b < e) {
    const uint64_t mid = b + (e - b) / 2;
    if (key[mid] < want) b = mid + 1; else e = mid;
  }
  return b;
}

// construction: this rank's edges [out[0], out[1]) are those whose lo is in [row_left, row_left + n_part)
__global__ void truss_range_kernel(const uint64_t* __restrict__ ekey, uint64_t m, uint32_t row_left, uint32_t n_part,
                                   uint64_t* __restrict__ out) {
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    out[0] = truss_lower_bound(ekey, 0, m, (uint64_t)row_left << 32);
    out[1] = truss_lower_bound(ekey, 0, m, ((uint64_t)row_left + n_part) << 32);
  }
}

// construction: the edge id of every oriented position (a warp per vertex u walks N+(u))
__global__ void truss_orient_ids_kernel(const uint64_t* __restrict__ off, const uint32_t* __restrict__ dst, uint32_t nv,
                                        const uint64_t* __restrict__ ekey, uint64_t m, uint32_t* __restrict__ eid) {
  const uint32_t warps = gridDim.x * (blockDim.x >> 5);
  for (uint32_t u = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); u < nv; u += warps)
    for (uint64_t j = off[u] + (threadIdx.x & 31); j < off[u + 1]; j += 32) {
      const uint32_t v = dst[j];
      eid[j] = (uint32_t)truss_lower_bound(ekey, 0, m, (uint64_t)min(u, v) << 32 | max(u, v));
    }
}

// construction: both directions of every edge, src << 32 | dst with the edge id as the sort value
__global__ void truss_emit_kernel(const uint64_t* __restrict__ ekey, uint64_t m, uint64_t* __restrict__ key, uint32_t* __restrict__ id) {
  for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < m; i += (uint64_t)gridDim.x * blockDim.x) {
    const uint64_t k = ekey[i];
    key[2 * i] = k;
    key[2 * i + 1] = k << 32 | k >> 32;
    id[2 * i] = id[2 * i + 1] = (uint32_t)i;
  }
}

// construction: sorted entries -> adjacency (neighbour << 32 | edge id) and list lengths
__global__ void truss_lists_kernel(const uint64_t* __restrict__ key, const uint32_t* __restrict__ id, uint64_t n,
                                   uint64_t* __restrict__ adj, uint32_t* __restrict__ len) {
  for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) {
    adj[i] = key[i] << 32 | id[i];
    atomicAdd(len + (uint32_t)(key[i] >> 32), 1u);
  }
}

// F marked dying, τ = ℓ + 2 on it (every rank marks the whole of F); the round's record cleared
__global__ void truss_mark_kernel(const uint32_t* __restrict__ f, uint32_t nf, uint32_t tau, uint8_t* __restrict__ st,
                                  uint32_t* __restrict__ truss, KcoreRec* __restrict__ rec) {
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < nf; i += gridDim.x * blockDim.x) {
    st[f[i]] = kTrussDying;
    truss[f[i]] = tau;
  }
  if (blockIdx.x == 0 && threadIdx.x == 0) *rec = KcoreRec{0, 0, 0, 0, kKcoreNoMin};
}

__global__ void truss_kill_kernel(const uint32_t* __restrict__ f, uint32_t nf, uint8_t* __restrict__ st) {
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < nf; i += gridDim.x * blockDim.x) st[f[i]] = kTrussDead;
}

// slots of every F edge: the length of the shorter of its two lists; 0 at [nf]
__global__ void truss_lengths_kernel(const uint32_t* __restrict__ f, uint32_t nf, const uint64_t* __restrict__ ekey,
                                     const uint64_t* __restrict__ off, uint64_t* __restrict__ pre) {
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i <= nf; i += gridDim.x * blockDim.x) {
    uint64_t n = 0;
    if (i < nf) {
      const uint64_t k = ekey[f[i]];
      const uint32_t u = (uint32_t)(k >> 32), v = (uint32_t)k;
      n = min(off[u + 1] - off[u], off[v + 1] - off[v]);
    }
    pre[i] = n;
  }
}

struct TrussWalkArgs {
  const uint32_t* f;      // [nf] the global F
  uint32_t nf;
  const uint64_t* pre;    // [nf + 1] exclusive scan of the slots; pre[nf] = slots of the round
  const uint64_t* ekey;   // [m] lo << 32 | hi
  const uint64_t* off;    // [nv + 1] symmetric adjacency offsets
  const uint64_t* adj;    // neighbour << 32 | edge id
  const uint8_t* st;      // [m] alive / dying / dead
  uint32_t* sup;          // [m] (this rank keeps its own edges' current)
  uint32_t e_lo, e_hi;    // this rank's edges [e_lo, e_hi)
  uint32_t l;             // ℓ = k - 2
  uint32_t* next;         // next piece
  KcoreRec* rec;          // next = appends; flag = 1 when a decrement found support 0
};

// One F edge's decrement of a triangle edge x it does not share with F: atomicSub, and the old value decides
__device__ __forceinline__ bool truss_lower(const TrussWalkArgs& a, uint32_t x) {
  const uint32_t old = atomicSub(a.sup + x, 1u);
  if (old == 0) atomicExch(&a.rec->flag, 1u);
  return old == a.l + 1;
}

// As kcore_scatter_kernel: every warp takes one contiguous range of the round's slots (a multiple of 32), finds the F
// edge of its first slot by one binary search and walks forward, so a hub's list is spread over every warp of the grid.
// Slot s of F edge e = {u, v} is entry s of the shorter list (of a), a neighbour w with the edge {a, w}, looked up in
// the list of the other endpoint b.
__global__ void __launch_bounds__(kTrussThreads) truss_walk_kernel(const __grid_constant__ TrussWalkArgs a) {
  const uint64_t total = a.pre[a.nf];
  const uint64_t warps = (uint64_t)gridDim.x * (blockDim.x >> 5);
  const uint64_t chunk = ((total + warps - 1) / warps + 31) & ~31ull;
  const uint64_t wi = (uint64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const uint64_t begin = wi * chunk;
  if (begin >= total) return;  // warp-uniform
  const uint64_t end = min(total, begin + chunk);
  uint32_t lo = 0, hi = a.nf - 1;  // last F edge with pre <= begin
  while (lo < hi) {
    const uint32_t mid = lo + (hi - lo + 1) / 2;
    if (a.pre[mid] <= begin) lo = mid; else hi = mid - 1;
  }
  uint32_t idx = lo;
  const int lane = threadIdx.x & 31;
  for (uint64_t s = begin; s < end; s += 32) {
    const uint64_t slot = s + lane;
    bool take1 = false, take2 = false;
    uint32_t e1 = 0, e2 = 0;
    if (slot < end) {
      while (a.pre[idx + 1] <= slot) ++idx;
      const uint32_t e = a.f[idx];
      const uint64_t k = a.ekey[e];
      uint32_t u = (uint32_t)(k >> 32), v = (uint32_t)k;
      if (a.off[v + 1] - a.off[v] < a.off[u + 1] - a.off[u]) { const uint32_t t = u; u = v; v = t; }  // u: the shorter list
      const uint64_t ent = a.adj[a.off[u] + (slot - a.pre[idx])];
      const uint32_t w = (uint32_t)(ent >> 32);
      e1 = (uint32_t)ent;  // {u, w}
      uint64_t b = a.off[v], en = a.off[v + 1];
      while (b < en) {
        const uint64_t mid = b + (en - b) / 2;
        if ((uint32_t)(a.adj[mid] >> 32) < w) b = mid + 1; else en = mid;
      }
      if (b < a.off[v + 1] && (uint32_t)(a.adj[b] >> 32) == w) {
        e2 = (uint32_t)a.adj[b];  // {v, w}
        const uint8_t s1 = a.st[e1], s2 = a.st[e2];
        const bool f1 = s1 == kTrussDying, f2 = s2 == kTrussDying;
        // the triangle counts iff no edge is dead; it is e's to apply iff e has the smallest id among its F edges
        if (s1 != kTrussDead && s2 != kTrussDead && !(f1 && e1 < e) && !(f2 && e2 < e)) {
          if (!f1 && e1 >= a.e_lo && e1 < a.e_hi) take1 = truss_lower(a, e1);
          if (!f2 && e2 >= a.e_lo && e2 < a.e_hi) take2 = truss_lower(a, e2);
        }
      }
    }
    kcore_append(take1, e1, &a.rec->next, a.next);
    kcore_append(take2, e2, &a.rec->next, a.next);
  }
}

// check: a warp per edge e of this rank, c = τ(e); over the common neighbours w, a = #(min(τ(u,w), τ(v,w)) >= c) and
// b = #(... >= c + 1); e violates iff c < 2, a < c - 2 or b >= c - 1
__global__ void truss_check_kernel(const uint64_t* __restrict__ ekey, uint32_t e_lo, uint32_t e_hi, const uint64_t* __restrict__ off,
                                   const uint64_t* __restrict__ adj, const uint32_t* __restrict__ truss,
                                   unsigned long long* __restrict__ bad) {
  const int lane = threadIdx.x & 31;
  const uint32_t warps = gridDim.x * (blockDim.x >> 5);
  uint32_t mine = 0;
  for (uint32_t e = e_lo + blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); e < e_hi; e += warps) {
    const uint64_t k = ekey[e];
    uint32_t u = (uint32_t)(k >> 32), v = (uint32_t)k;
    if (off[v + 1] - off[v] < off[u + 1] - off[u]) { const uint32_t t = u; u = v; v = t; }
    const uint64_t c = truss[e];
    uint32_t na = 0, nb = 0;
    for (uint64_t j = off[u] + lane; j < off[u + 1]; j += 32) {
      const uint64_t ent = adj[j];
      const uint32_t w = (uint32_t)(ent >> 32);
      uint64_t b = off[v], en = off[v + 1];
      while (b < en) {
        const uint64_t mid = b + (en - b) / 2;
        if ((uint32_t)(adj[mid] >> 32) < w) b = mid + 1; else en = mid;
      }
      if (b < off[v + 1] && (uint32_t)(adj[b] >> 32) == w) {
        const uint64_t t = min(truss[(uint32_t)ent], truss[(uint32_t)adj[b]]);
        na += t >= c;
        nb += t >= c + 1;
      }
    }
    for (int o = 16; o; o >>= 1) {
      na += __shfl_xor_sync(0xffffffffu, na, o);
      nb += __shfl_xor_sync(0xffffffffu, nb, o);
    }
    if (lane == 0) mine += c < 2 || (uint64_t)na + 2 < c || (uint64_t)nb + 1 >= c;
  }
  if (lane == 0 && mine) atomicAdd(bad, (unsigned long long)mine);
}

// tv[v] = max τ over the edges at v (tv zeroed by the caller)
__global__ void truss_vertex_kernel(const uint64_t* __restrict__ ekey, uint64_t m, const uint32_t* __restrict__ truss,
                                    uint32_t* __restrict__ tv) {
  for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < m; i += (uint64_t)gridDim.x * blockDim.x) {
    atomicMax(tv + (uint32_t)(ekey[i] >> 32), truss[i]);
    atomicMax(tv + (uint32_t)ekey[i], truss[i]);
  }
}

}  // namespace luxb
