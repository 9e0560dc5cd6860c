// tc.cuh — triangle counting (no reference counterpart), the kernels behind luxb_tc_run.
// The CSC's directed edges are read as an undirected simple graph: {u, v} is an edge iff u != v and u -> v or v -> u is
// stored (parallel edges, both directions and self-loops collapse; weights are ignored).
//
// Construction (luxb_init, once):
//   keys          : min << 32 | max per stored edge with u != v, radix sort + unique -> the m undirected edges
//   orientation   : each edge goes from the lower to the higher of (degree, id); sorted again -> CSR of the out-lists
//                   N+(u), ids ascending inside each list.  Degree order bounds |N+(u)| by sqrt(2m)
//   work          : W(u) = sum of |N+(v)| over v in N+(u), the probes u costs
//   bins          : u with 0 < |N+(u)| <= kTcSharedList are cut into groups of consecutive staged vertices (each group
//                   stages fewer than 2 kTcSharedList list entries and closes once it passes a multiple of kTcGroupProbes
//                   probes); u with a longer list is a "big" vertex, one CTA each; u with an empty list is skipped
// Counting (luxb_tc_run): every triangle a < b < c in that order is found once, at the oriented edge (a, b), as
// c in N+(a) ∩ N+(b).  The grouped kernel stages the out-lists of its vertices in shared memory with one counter per
// entry and flattens the probes of the whole group, sum over v of |N+(v)|, over all lanes, so a vertex whose lists are
// short does not leave most of a warp idle.  A probe looks w up in its owner's staged list by binary search; a hit adds
// one to the counters of w's and v's entries and to the owner's.  Counters go to t[] once per group and entry: no
// global atomic per triangle (the hubs rank highest and are the w of most triangles).  The big kernel stages its list
// in kTcSharedList-entry chunks and runs a warp per v of the list against each chunk.  Integers only: the result does
// not depend on the schedule.  Both kernels are templates on where the counts go (TcVertexSink here; k-truss counts
// edge support with the same kernels, truss.cuh).
#pragma once
#include <stdint.h>
#include <cuda_runtime.h>
#include <cub/block/block_scan.cuh>
#include "common.cuh"

namespace luxb {

constexpr uint32_t kTcSharedList = 1024;         // longest out-list staged whole; the big kernel's chunk
constexpr uint32_t kTcStage = 2 * kTcSharedList; // staged entries of a group: < kTcSharedList before its last vertex
constexpr uint64_t kTcGroupProbes = 1ull << 15;  // probes (+ staged entries) after which a group closes
constexpr int kTcThreads = 256;

// u before v in the orientation order: (undirected degree, id) ascending
__device__ __forceinline__ bool tc_before(uint32_t du, uint32_t u, uint32_t dv, uint32_t v) {
  return du < dv || (du == dv && u < v);
}

// one key min << 32 | max per in-edge (u -> v) of this rank's CSC slice with u != v, compacted through `cursor`
__global__ void tc_emit_keys_kernel(const uint64_t* __restrict__ row_end_rel, uint32_t n_part, uint64_t e_part, uint32_t row_left,
                                    const uint32_t* __restrict__ src, unsigned long long* __restrict__ cursor,
                                    uint64_t* __restrict__ keys) {
  const uint32_t lane = threadIdx.x & 31;
  const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
  for (uint64_t base = (uint64_t)blockIdx.x * blockDim.x + (threadIdx.x & ~31u); base < e_part; base += stride) {
    const uint64_t e = base + lane;
    uint64_t key = 0;
    bool ok = false;
    if (e < e_part) {
      uint32_t lo = 0, hi = n_part;  // first row with row_end_rel > e
      while (lo < hi) {
        const uint32_t mid = lo + (hi - lo) / 2;
        if (row_end_rel[mid] > e) hi = mid; else lo = mid + 1;
      }
      const uint32_t v = row_left + lo, u = src[e];
      ok = u != v;
      key = (uint64_t)min(u, v) << 32 | max(u, v);
    }
    const uint32_t mask = __ballot_sync(0xFFFFFFFFu, ok);
    unsigned long long at = 0;
    if (lane == 0 && mask) at = atomicAdd(cursor, (unsigned long long)__popc(mask));
    at = __shfl_sync(0xFFFFFFFFu, at, 0);
    if (ok) keys[at + __popc(mask & ((1u << lane) - 1u))] = key;
  }
}

// undirected degree of every vertex from the unique edge keys
__global__ void tc_degree_kernel(const uint64_t* __restrict__ keys, uint64_t m, uint32_t* __restrict__ deg) {
  for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < m; i += (uint64_t)gridDim.x * blockDim.x) {
    atomicAdd(deg + (uint32_t)(keys[i] >> 32), 1u);
    atomicAdd(deg + (uint32_t)keys[i], 1u);
  }
}

// orient every edge (in place: from << 32 | to) and count the out-degrees
__global__ void tc_orient_kernel(uint64_t* __restrict__ keys, uint64_t m, const uint32_t* __restrict__ deg, uint32_t* __restrict__ outdeg) {
  for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < m; i += (uint64_t)gridDim.x * blockDim.x) {
    const uint32_t a = (uint32_t)(keys[i] >> 32), b = (uint32_t)keys[i];
    const bool ab = tc_before(deg[a], a, deg[b], b);
    const uint32_t from = ab ? a : b, to = ab ? b : a;
    keys[i] = (uint64_t)from << 32 | to;
    atomicAdd(outdeg + from, 1u);
  }
}

// sorted oriented keys -> out-list ids, and W(u) += |N+(v)| for every oriented edge (u, v)
__global__ void tc_lists_kernel(const uint64_t* __restrict__ keys, uint64_t m, const uint64_t* __restrict__ off, uint32_t* __restrict__ dst,
                                unsigned long long* __restrict__ work) {
  for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < m; i += (uint64_t)gridDim.x * blockDim.x) {
    const uint32_t u = (uint32_t)(keys[i] >> 32), v = (uint32_t)keys[i];
    dst[i] = v;
    atomicAdd(work + u, (unsigned long long)(off[v + 1] - off[v]));
  }
}

// vertices of the grouped kernel, and the big ones
struct TcStaged {
  const uint64_t* off;
  __device__ bool operator()(uint32_t u) const {
    const uint64_t d = off[u + 1] - off[u];
    return d > 0 && d <= kTcSharedList;
  }
};
struct TcBig {
  const uint64_t* off;
  __device__ bool operator()(uint32_t u) const { return off[u + 1] - off[u] > kTcSharedList; }
};

// per staged vertex k: its list length and its cost (probes + list), scanned exclusively afterwards ([n] = 0)
__global__ void tc_cost_kernel(const uint32_t* __restrict__ staged, uint32_t n, const uint64_t* __restrict__ off,
                               const unsigned long long* __restrict__ work, uint64_t* __restrict__ len, uint64_t* __restrict__ cost) {
  for (uint64_t k = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; k <= n; k += (uint64_t)gridDim.x * blockDim.x) {
    uint64_t d = 0, c = 0;
    if (k < n) {
      const uint32_t u = staged[k];
      d = off[u + 1] - off[u];
      c = work[u] + d;
    }
    len[k] = d;
    cost[k] = c;
  }
}

// a group starts where the staged-entry prefix crosses a multiple of kTcSharedList or the cost prefix one of
// kTcGroupProbes: all but the last vertex of a group then stage fewer than kTcSharedList entries together
struct TcGroupHead {
  const uint64_t* len_pre;
  const uint64_t* cost_pre;
  __device__ bool operator()(uint32_t k) const {
    return k == 0 || len_pre[k] / kTcSharedList != len_pre[k - 1] / kTcSharedList ||
           cost_pre[k] / kTcGroupProbes != cost_pre[k - 1] / kTcGroupProbes;
  }
};

struct TcArgs {
  const uint64_t* off;         // [nv + 1] oriented CSR offsets
  const uint32_t* dst;         // N+(u) ids, ascending inside each list
  const uint32_t* staged;      // [n_staged] vertices of this rank's range with 0 < |N+| <= kTcSharedList, ascending
  const uint64_t* stage_pre;   // [n_staged + 1] exclusive prefix of their list lengths
  const uint32_t* group;       // [n_group + 1] first staged index of every group, then n_staged
  uint32_t n_group;
  const uint32_t* big;         // [n_big] vertices of this rank's range with |N+| > kTcSharedList
  uint32_t n_big;
  unsigned long long* t;       // [nv] per-vertex triangle counts
  unsigned int* next;          // [2] work counters (groups, big vertices), zero at launch
};

// Where the grouped and big kernels send what they count.  TcVertexSink: triangles per vertex into a.t (the owner's
// share from s_own).  TrussEdgeSink (truss.cuh): support per edge, sup[eid[p]] for the oriented position p of each
// edge of a triangle; no per-vertex share.
struct TcVertexSink {
  static constexpr bool kPerEdge = false;
};

template <class Sink>
__device__ __forceinline__ void tc_group_body(const TcArgs& a, const Sink& sink) {
  typedef cub::BlockScan<uint32_t, kTcThreads> Scan;
  constexpr int kPer = kTcStage / kTcThreads;
  __shared__ uint32_t s_id[kTcStage];        // staged ids: the lists of the group's vertices, back to back
  __shared__ uint32_t s_cnt[kTcStage];       // triangles found at each entry (as w or as v)
  __shared__ uint32_t s_pre[kTcStage + 1];   // exclusive prefix of |N+(id)|: probe k belongs to the entry j with pre[j] <= k < pre[j + 1]
  __shared__ uint32_t s_own[kTcStage];       // triangles of each group vertex (as u)
  __shared__ uint16_t s_q[kTcStage];         // owner (group-local vertex) of each entry
  __shared__ uint16_t s_sp[kTcStage + 1];    // owner q's entries are [sp[q], sp[q + 1])
  __shared__ typename Scan::TempStorage s_scan;
  __shared__ uint32_t s_g;
  const uint32_t tid = threadIdx.x;
  for (;;) {
    if (tid == 0) s_g = atomicAdd(a.next, 1u);
    __syncthreads();
    const uint32_t gi = s_g;
    if (gi >= a.n_group) break;
    const uint32_t k0 = a.group[gi], nq = a.group[gi + 1] - k0;
    const uint64_t e0 = a.stage_pre[k0];
    const uint32_t S = (uint32_t)(a.stage_pre[k0 + nq] - e0);
    for (uint32_t q = tid; q <= nq; q += kTcThreads) s_sp[q] = (uint16_t)(a.stage_pre[k0 + q] - e0);
    for (uint32_t q = tid; q < nq; q += kTcThreads) s_own[q] = 0;
    __syncthreads();
    for (uint32_t i = tid; i < S; i += kTcThreads) {
      uint32_t lo = 0, hi = nq;  // owner: last q with sp[q] <= i
      while (hi - lo > 1) {
        const uint32_t mid = (lo + hi) / 2;
        if (s_sp[mid] <= i) lo = mid; else hi = mid;
      }
      const uint32_t u = a.staged[k0 + lo];
      const uint32_t v = a.dst[a.off[u] + (i - s_sp[lo])];
      s_id[i] = v;
      s_q[i] = (uint16_t)lo;
      s_cnt[i] = 0;
      s_pre[i] = (uint32_t)(a.off[v + 1] - a.off[v]);
    }
    __syncthreads();
    uint32_t len[kPer];
#pragma unroll
    for (int r = 0; r < kPer; ++r) len[r] = tid * kPer + r < S ? s_pre[tid * kPer + r] : 0u;
    uint32_t total;
    Scan(s_scan).ExclusiveSum(len, len, total);
#pragma unroll
    for (int r = 0; r < kPer; ++r) if (tid * kPer + r < S) s_pre[tid * kPer + r] = len[r];
    if (tid == 0) s_pre[S] = total;
    __syncthreads();
    // the probes of the whole group, flattened: consecutive lanes read consecutive ids of one list.  A thread's probes
    // ascend, so its entry j and owner q only ascend: their hits are added in runs
    uint32_t run_j = 0, run_c = 0, run_q = 0, run_o = 0;
    for (uint32_t k = tid; k < total; k += kTcThreads) {
      uint32_t lo = 0, hi = S;  // entry: last j with pre[j] <= k
      while (hi - lo > 1) {
        const uint32_t mid = (lo + hi) / 2;
        if (s_pre[mid] <= k) lo = mid; else hi = mid;
      }
      const uint32_t j = lo, q = s_q[j], v = s_id[j];
      const uint32_t w = __ldg(a.dst + a.off[v] + (k - s_pre[j]));
      const uint32_t end = s_sp[q + 1];
      uint32_t b = s_sp[q], e = end;
      while (b < e) {
        const uint32_t mid = (b + e) / 2;
        if (s_id[mid] < w) b = mid + 1; else e = mid;
      }
      if (b < end && s_id[b] == w) {
        atomicAdd(&s_cnt[b], 1u);
        if (j != run_j) {
          if (run_c) atomicAdd(&s_cnt[run_j], run_c);
          run_j = j;
          run_c = 0;
        }
        ++run_c;
        if constexpr (Sink::kPerEdge) {
          sink.add(a.off[v] + (k - s_pre[j]), 1u);  // the edge (v, w)
        } else {
          if (q != run_q) {
            if (run_o) atomicAdd(&s_own[run_q], run_o);
            run_q = q;
            run_o = 0;
          }
          ++run_o;
        }
      }
    }
    if (run_c) atomicAdd(&s_cnt[run_j], run_c);
    if constexpr (!Sink::kPerEdge) {
      if (run_o) atomicAdd(&s_own[run_q], run_o);
    }
    __syncthreads();
    if constexpr (Sink::kPerEdge) {  // entry i is the edge (owner, s_id[i])
      for (uint32_t i = tid; i < S; i += kTcThreads)
        if (s_cnt[i]) sink.add(a.off[a.staged[k0 + s_q[i]]] + (i - s_sp[s_q[i]]), s_cnt[i]);
    } else {
      for (uint32_t i = tid; i < S; i += kTcThreads)
        if (s_cnt[i]) atomicAdd(a.t + s_id[i], (unsigned long long)s_cnt[i]);
      for (uint32_t q = tid; q < nq; q += kTcThreads)
        if (s_own[q]) atomicAdd(a.t + a.staged[k0 + q], (unsigned long long)s_own[q]);
    }
    __syncthreads();  // shared memory is restaged by the next group
  }
}

__global__ void __launch_bounds__(kTcThreads) tc_group_kernel(const __grid_constant__ TcArgs a) { tc_group_body(a, TcVertexSink{}); }

// one CTA per big vertex u: N+(u) staged kTcSharedList entries at a time; a warp per v in N+(u) probes N+(v) against
// the chunk.  c(u, v) goes to t[v] once per chunk and v, the chunk's counters to t[w], the sum of c to t[u]
template <class Sink>
__device__ __forceinline__ void tc_big_body(const TcArgs& a, const Sink& sink) {
  __shared__ uint32_t s_id[kTcSharedList];
  __shared__ uint32_t s_cnt[kTcSharedList];
  __shared__ unsigned long long s_own;
  __shared__ uint32_t s_b;
  const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  for (;;) {
    if (tid == 0) { s_b = atomicAdd(a.next + 1, 1u); s_own = 0; }
    __syncthreads();
    const uint32_t bi = s_b;
    if (bi >= a.n_big) break;
    const uint32_t u = a.big[bi];
    const uint64_t ub = a.off[u];
    const uint32_t du = (uint32_t)(a.off[u + 1] - ub);
    unsigned long long own = 0;
    for (uint32_t c0 = 0; c0 < du; c0 += kTcSharedList) {
      const uint32_t cn = min(kTcSharedList, du - c0);
      for (uint32_t i = tid; i < cn; i += kTcThreads) {
        s_id[i] = a.dst[ub + c0 + i];
        s_cnt[i] = 0;
      }
      __syncthreads();
      const uint32_t first = s_id[0], last = s_id[cn - 1];
      for (uint32_t j = warp; j < du; j += kTcThreads / 32) {
        const uint32_t v = a.dst[ub + j];
        const uint64_t vb = a.off[v];
        const uint32_t vn = (uint32_t)(a.off[v + 1] - vb);
        uint32_t c = 0;
        for (uint32_t p = lane; p < vn; p += 32) {
          const uint32_t w = __ldg(a.dst + vb + p);
          if (w > last) break;  // the list ascends: nothing further is in this chunk
          if (w < first) continue;
          uint32_t b = 0, e = cn;
          while (b < e) {
            const uint32_t mid = (b + e) / 2;
            if (s_id[mid] < w) b = mid + 1; else e = mid;
          }
          if (b < cn && s_id[b] == w) {
            atomicAdd(&s_cnt[b], 1u);
            ++c;
            if constexpr (Sink::kPerEdge) sink.add(vb + p, 1u);  // the edge (v, w)
          }
        }
#pragma unroll
        for (int o = 16; o; o >>= 1) c += __shfl_xor_sync(0xFFFFFFFFu, c, o);
        if (lane == 0 && c) {
          if constexpr (Sink::kPerEdge) {
            sink.add(ub + j, c);  // the edge (u, v)
          } else {
            atomicAdd(a.t + v, (unsigned long long)c);
            own += c;
          }
        }
      }
      __syncthreads();
      for (uint32_t i = tid; i < cn; i += kTcThreads) {
        if constexpr (Sink::kPerEdge) {
          if (s_cnt[i]) sink.add(ub + c0 + i, s_cnt[i]);  // the edge (u, w)
        } else {
          if (s_cnt[i]) atomicAdd(a.t + s_id[i], (unsigned long long)s_cnt[i]);
        }
      }
      __syncthreads();  // the next chunk overwrites s_id / s_cnt
    }
    if constexpr (!Sink::kPerEdge) {
      if (own) atomicAdd(&s_own, own);
      __syncthreads();
      if (tid == 0 && s_own) atomicAdd(a.t + u, s_own);
    }
    __syncthreads();  // s_own / s_b are reset for the next vertex
  }
}

__global__ void __launch_bounds__(kTcThreads) tc_big_kernel(const __grid_constant__ TcArgs a) { tc_big_body(a, TcVertexSink{}); }

}  // namespace luxb
