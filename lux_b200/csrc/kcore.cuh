// kcore.cuh — k-core decomposition (no reference counterpart), the kernels behind luxb_kcore_run.
// The graph is LUXB_TC's: the CSC's directed edges read as an undirected simple graph.  core[v] is the largest k such
// that v lies in a subgraph whose every vertex has degree >= k.
//
// Construction (luxb_init, once): the distinct undirected keys of the whole graph (shared with TC), then this rank's
// adjacency: for every key {a, b} the entry a -> b if b is this rank's and b -> a if a is, sorted by (src, dst) into a
// CSR over all nv sources whose targets are this rank's vertices.  Every adjacency entry of the graph is held by exactly
// one rank (2m in all); this rank's deg(v) is the number of entries that target v.
//
// The peel (luxb_kcore_run), level-synchronous:
//   k = 0; while a vertex is alive: k = max(k, min deg over alive vertices); repeat: F = {alive v : deg(v) <= k}; stop if
//   F is empty; core[F] = k, remove F, lower the degrees of the remaining vertices.
// A round is one non-empty F.  Per round, on every rank: mark core = k on this rank's piece of F (before the scatter,
// so that members of F never decrement each other); the pieces are exchanged; the adjacency entries this rank holds for
// the global F are flattened (an exclusive scan of the list lengths) and spread over the whole grid, each warp taking a
// contiguous slot range from one binary search and walking forward; every alive target u takes
// old = atomicSub(&deg[u], 1) and, iff old == k + 1, joins the next piece (the crossing happens once per u: exactly-once
// enqueue, warp-aggregated).  Where this rank's next piece is empty, the tally then compacts the alive list and reduces
// (alive count, min deg, count at the min), which tells the host both whether the level goes on and, if not, the sizes of the next level's first pieces
// (the alive vertices with deg == the new k).  Integers only; only the order inside a piece depends on the schedule.
#pragma once
#include <stdint.h>
#include <cuda_runtime.h>
#include "common.cuh"

namespace luxb {

constexpr uint32_t kKcoreUnset = 0xFFFFFFFFu;  // core of a vertex still alive during a run
constexpr int kKcoreThreads = 256;

// per-rank record of a round, read by the host once per round (all-gathered on several ranks)
struct KcoreRec {
  uint32_t next;                 // this rank's next piece (scatter appends)
  uint32_t alive;                // this rank's alive vertices after the round (tally appends)
  uint32_t sel;                  // appends of the level-start select
  uint32_t flag;                 // LUXB_TRUSS (truss.cuh): set when a decrement found support 0
  unsigned long long min_cnt;    // min deg << 32 | number of alive vertices at that deg (kKcoreNoMin when none alive)
};
constexpr unsigned long long kKcoreNoMin = 0xFFFFFFFF00000000ull;

__device__ __forceinline__ unsigned long long kcore_min_combine(unsigned long long a, unsigned long long b) {
  const uint32_t ma = (uint32_t)(a >> 32), mb = (uint32_t)(b >> 32);
  if (ma != mb) return ma < mb ? a : b;
  return a + (uint32_t)b;  // same min: counts add (never carries: at most nv alive vertices)
}

// warp-aggregated append of v (where `take`) through `cursor`; every lane of the warp calls it
__device__ __forceinline__ void kcore_append(bool take, uint32_t v, uint32_t* cursor, uint32_t* out) {
  const int lane = threadIdx.x & 31;
  const unsigned m = __ballot_sync(0xffffffffu, take);
  if (!m) return;
  const int leader = __ffs(m) - 1;
  uint32_t pos = 0;
  if (lane == leader) pos = atomicAdd(cursor, (uint32_t)__popc(m));
  pos = __shfl_sync(0xffffffffu, pos, leader);
  if (take) out[pos + __popc(m & ((1u << lane) - 1u))] = v;
}

// construction: this rank's entries src << 32 | dst (dst in [row_left, row_right]) of every undirected key; with
// out == nullptr only their number (cursor)
__global__ void kcore_emit_kernel(const uint64_t* __restrict__ keys, uint64_t m, uint32_t row_left, uint32_t row_right,
                                  unsigned long long* __restrict__ cursor, uint64_t* __restrict__ out) {
  const uint32_t lane = threadIdx.x & 31;
  const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
  for (uint64_t base = (uint64_t)blockIdx.x * blockDim.x + (threadIdx.x & ~31u); base < m; base += stride) {
    const uint64_t i = base + lane;
    uint32_t a = 0, b = 0;
    if (i < m) { a = (uint32_t)(keys[i] >> 32); b = (uint32_t)keys[i]; }
    const bool ab = i < m && b >= row_left && b <= row_right;  // a -> b, b this rank's
    const bool ba = i < m && a >= row_left && a <= row_right;  // b -> a
    const uint32_t mab = __ballot_sync(0xFFFFFFFFu, ab), mba = __ballot_sync(0xFFFFFFFFu, ba);
    unsigned long long at = 0;
    if (lane == 0 && (mab | mba)) at = atomicAdd(cursor, (unsigned long long)(__popc(mab) + __popc(mba)));
    at = __shfl_sync(0xFFFFFFFFu, at, 0);
    const uint32_t below = (1u << lane) - 1u;
    if (!out) continue;
    if (ab) out[at + __popc(mab & below)] = (uint64_t)a << 32 | b;
    if (ba) out[at + __popc(mab) + __popc(mba & below)] = (uint64_t)b << 32 | a;
  }
}

// construction: sorted entries -> adjacency ids, list lengths per source, this rank's degrees
__global__ void kcore_lists_kernel(const uint64_t* __restrict__ entries, uint64_t n, uint32_t row_left, uint32_t* __restrict__ adj,
                                   uint32_t* __restrict__ len, uint32_t* __restrict__ deg) {
  for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) {
    const uint32_t src = (uint32_t)(entries[i] >> 32), dst = (uint32_t)entries[i];
    adj[i] = dst;
    atomicAdd(len + src, 1u);
    atomicAdd(deg + (dst - row_left), 1u);
  }
}

// run start: every own vertex alive (core unset, deg from the construction, on the alive list), the record cleared
__global__ void kcore_reset_kernel(uint32_t* __restrict__ core, uint32_t* __restrict__ deg, const uint32_t* __restrict__ deg0,
                                   uint32_t* __restrict__ alive, uint32_t n_part, uint32_t row_left, KcoreRec* __restrict__ rec) {
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n_part; i += gridDim.x * blockDim.x) {
    core[row_left + i] = kKcoreUnset;
    deg[i] = deg0[i];
    alive[i] = row_left + i;
  }
  if (blockIdx.x == 0 && threadIdx.x == 0) *rec = KcoreRec{0, 0, 0, 0, kKcoreNoMin};
}

// compact the alive list (core still unset) and reduce alive count, min deg and the count at the min into the record.
// Skipped (the list stays as it was) when the scatter appended to this rank's next piece: then the global next F is not
// empty either, the level goes on, and the host needs neither the min nor the compacted list.  A level therefore ends
// only after a round in which every rank ran the tally.
__global__ void __launch_bounds__(kKcoreThreads) kcore_tally_kernel(const uint32_t* __restrict__ alive_in, uint32_t n_alive,
                                                                     const uint32_t* __restrict__ core, const uint32_t* __restrict__ deg,
                                                                     uint32_t row_left, uint32_t* __restrict__ alive_out,
                                                                     KcoreRec* __restrict__ rec) {
  __shared__ unsigned long long s_warp[kKcoreThreads / 32];
  if (*(volatile uint32_t*)&rec->next) return;  // whole CTA
  unsigned long long mc = kKcoreNoMin;
  const uint32_t stride = gridDim.x * blockDim.x;
  for (uint32_t base = blockIdx.x * blockDim.x + (threadIdx.x & ~31u); base < n_alive; base += stride) {
    const uint32_t i = base + (threadIdx.x & 31);
    uint32_t v = 0;
    bool live = false;
    if (i < n_alive) {
      v = alive_in[i];
      live = core[v] == kKcoreUnset;
      if (live) mc = kcore_min_combine(mc, (unsigned long long)deg[v - row_left] << 32 | 1u);
    }
    kcore_append(live, v, &rec->alive, alive_out);
  }
  for (int o = 16; o; o >>= 1) mc = kcore_min_combine(mc, __shfl_xor_sync(0xffffffffu, mc, o));
  if ((threadIdx.x & 31) == 0) s_warp[threadIdx.x >> 5] = mc;
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int w = 1; w < kKcoreThreads / 32; ++w) mc = kcore_min_combine(mc, s_warp[w]);
    if (mc != kKcoreNoMin) {  // one compare-and-swap loop per CTA
      unsigned long long seen = rec->min_cnt;
      for (;;) {
        const unsigned long long want = kcore_min_combine(seen, mc);
        if (want == seen) break;
        const unsigned long long got = atomicCAS(&rec->min_cnt, seen, want);
        if (got == seen) break;
        seen = got;
      }
    }
  }
}

// level start: the alive vertices with deg == k form this rank's first piece of the level
__global__ void kcore_select_kernel(const uint32_t* __restrict__ alive, uint32_t n_alive, const uint32_t* __restrict__ deg,
                                    uint32_t row_left, uint32_t k, uint32_t* __restrict__ piece, KcoreRec* __restrict__ rec) {
  for (uint32_t base = blockIdx.x * blockDim.x + (threadIdx.x & ~31u); base < n_alive; base += gridDim.x * blockDim.x) {
    const uint32_t i = base + (threadIdx.x & 31);
    const uint32_t v = i < n_alive ? alive[i] : 0;
    kcore_append(i < n_alive && deg[v - row_left] == k, v, &rec->sel, piece);
  }
}

// core = k on this rank's piece of F, before any decrement of the round; the round's record cleared
__global__ void kcore_mark_kernel(const uint32_t* __restrict__ piece, uint32_t n, uint32_t k, uint32_t* __restrict__ core,
                                  KcoreRec* __restrict__ rec) {
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) core[piece[i]] = k;
  if (blockIdx.x == 0 && threadIdx.x == 0) *rec = KcoreRec{0, 0, 0, 0, kKcoreNoMin};
}

// lengths of this rank's lists of the global F (scanned in place into slot offsets by the caller), 0 at [nF]
__global__ void kcore_lengths_kernel(const uint32_t* __restrict__ f, uint32_t nf, const uint64_t* __restrict__ off,
                                     uint64_t* __restrict__ pre) {
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i <= nf; i += gridDim.x * blockDim.x)
    pre[i] = i < nf ? off[f[i] + 1] - off[f[i]] : 0;
}

struct KcoreScatterArgs {
  const uint32_t* f;     // [nf] the global F
  uint32_t nf;
  const uint64_t* pre;   // [nf + 1] exclusive scan of this rank's list lengths; pre[nf] = slots of the round
  const uint64_t* off;   // [nv + 1] adjacency offsets
  const uint32_t* adj;
  const uint32_t* core;  // kKcoreUnset = alive
  uint32_t* deg;         // [n_part]
  uint32_t row_left;
  uint32_t k;
  uint32_t* next;        // next piece
  KcoreRec* rec;
};

// Every warp takes one contiguous range of the round's slots (a multiple of 32), finds the F entry of its first slot by
// one binary search and walks forward: lane l handles slots begin + l, begin + l + 32, ..., so a hub's list is spread
// over every warp of the grid and a run of short lists fills every lane.
__global__ void __launch_bounds__(kKcoreThreads) kcore_scatter_kernel(const __grid_constant__ KcoreScatterArgs a) {
  const uint64_t total = a.pre[a.nf];
  const uint64_t warps = (uint64_t)gridDim.x * (blockDim.x >> 5);
  const uint64_t chunk = ((total + warps - 1) / warps + 31) & ~31ull;
  const uint64_t w = (uint64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const uint64_t begin = w * chunk;
  if (begin >= total) return;  // warp-uniform
  const uint64_t end = min(total, begin + chunk);
  uint32_t lo = 0, hi = a.nf - 1;  // last entry with pre <= begin (lists of length 0 share their pre with the next one)
  while (lo < hi) {
    const uint32_t mid = lo + (hi - lo + 1) / 2;
    if (a.pre[mid] <= begin) lo = mid; else hi = mid - 1;
  }
  uint32_t idx = lo;
  const int lane = threadIdx.x & 31;
  for (uint64_t s = begin; s < end; s += 32) {
    const uint64_t slot = s + lane;
    bool take = false;
    uint32_t u = 0;
    if (slot < end) {
      while (a.pre[idx + 1] <= slot) ++idx;
      const uint32_t v = a.f[idx];
      u = a.adj[a.off[v] + (slot - a.pre[idx])];
      if (a.core[u] == kKcoreUnset) take = atomicSub(a.deg + (u - a.row_left), 1u) == a.k + 1;
    }
    kcore_append(take, u, &a.rec->next, a.next);
  }
}

// check, pass 1: for every entry u -> v this rank holds, cnt[v] += (core[u] >= core[v]), cnt[n_part + v] += (core[u] > core[v])
__global__ void kcore_check_count_kernel(const uint64_t* __restrict__ off, const uint32_t* __restrict__ adj, uint32_t nv,
                                         const uint32_t* __restrict__ core, uint32_t row_left, uint32_t n_part,
                                         uint32_t* __restrict__ cnt) {
  const int lane = threadIdx.x & 31;
  const uint32_t warps = gridDim.x * (blockDim.x >> 5);
  for (uint32_t u = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); u < nv; u += warps) {
    const uint32_t cu = core[u];
    for (uint64_t j = off[u] + lane; j < off[u + 1]; j += 32) {
      const uint32_t v = adj[j], cv = core[v];
      if (cu >= cv) atomicAdd(cnt + (v - row_left), 1u);
      if (cu > cv) atomicAdd(cnt + n_part + (v - row_left), 1u);
    }
  }
}

// check, pass 2: v with c = core[v] violates the h-index fixpoint iff a < c or b >= c + 1
__global__ void kcore_check_kernel(const uint32_t* __restrict__ core, uint32_t row_left, uint32_t n_part, const uint32_t* __restrict__ cnt,
                                   unsigned long long* __restrict__ bad) {
  uint32_t mine = 0;
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n_part; i += gridDim.x * blockDim.x) {
    const uint64_t c = core[row_left + i];
    mine += (uint64_t)cnt[i] < c || (uint64_t)cnt[n_part + i] >= c + 1;
  }
  for (int o = 16; o; o >>= 1) mine += __shfl_xor_sync(0xffffffffu, mine, o);
  if ((threadIdx.x & 31) == 0 && mine) atomicAdd(bad, (unsigned long long)mine);
}

}  // namespace luxb
