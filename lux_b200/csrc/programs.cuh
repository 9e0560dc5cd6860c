// programs.cuh — the vertex-program surface (init / compute / update) that Lux leaves implicit in its kernels
// (SURVEY §8b "Vertex program").  Each struct mirrors one app.h + the arithmetic of its *_gpu.cu:
//   PageRankProgram : pagerank/app.h:19-35,   pagerank_gpu.cu:86-100 (compute+update), :255-259 (init)
//   MaxLabelProgram : components/app.h:19-38, components_gpu.cu:112-122 (pull), :48-82 (push), :738-739 (init)
//   HopDistProgram  : sssp/app.h,             sssp_gpu.cu:112-122, :57-59,75-77, :733-744 (init, INF = nv)
//   WeightedDistProgram: weighted SSSP over the CSC's i32 weights (ours; the reference has none)
// Kernels are templated on these; adding an app = adding a struct.  kWeighted programs take the edge weight in
// gather(src_val, w); every branch on it is `if constexpr`, so the unweighted instantiations are unchanged.
#pragma once
#include <stdint.h>
#include <cuda_runtime.h>

#ifndef LUXB_MAX_PEERS
#define LUXB_MAX_PEERS 63
#endif

namespace luxb {

constexpr float kAlpha = 0.15f;  // ALPHA, pagerank/app.h:24

struct PageRankProgram {
  using Vertex = float;  // stored value = rank / out-degree (pagerank_gpu.cu:98-100)
  using Acc = float;
  using Wide = double;
  struct Params {
    float init_rank;      // (1 - ALPHA) / nv, pagerank_gpu.cu:144
    const uint32_t* deg;  // global out-degrees (pull_scan_task_impl, pull_model.inl:333-343)
  };
  static constexpr bool kNeedsOld = false;
  static constexpr bool kWeighted = false;
  __device__ __forceinline__ static Acc identity() { return 0.0f; }
  __device__ __forceinline__ static Acc gather(Vertex src_val) { return src_val; }
  __device__ __forceinline__ static Acc combine(Acc x, Acc y) { return x + y; }
  __device__ __forceinline__ static Wide widen(Acc x) { return (double)x; }
  __device__ __forceinline__ static Wide wcombine(Wide x, Wide y) { return x + y; }
  __device__ __forceinline__ static Acc narrow(Wide x) { return (float)x; }
  __device__ __forceinline__ static Vertex update(uint32_t v, Acc acc, Vertex, const Params& p) {
    float y = __fmaf_rn(kAlpha, acc, p.init_rank);
    uint32_t d = __ldg(p.deg + v);
    return d != 0 ? __fdiv_rn(y, (float)d) : y;
  }
};

struct MaxLabelProgram {  // connected components: label = max id that reaches the vertex
  using Vertex = uint32_t;
  using Acc = uint32_t;
  using Wide = uint32_t;
  struct Params { uint32_t unused; };
  static constexpr bool kNeedsOld = true;  // new = max(old, gathered)  (components_gpu.cu:106)
  static constexpr bool kIsMax = true;
  static constexpr bool kWeighted = false;
  __device__ __forceinline__ static Acc identity() { return 0u; }
  __device__ __forceinline__ static Acc gather(Vertex src_val) { return src_val; }
  __device__ __forceinline__ static Acc combine(Acc x, Acc y) { return x > y ? x : y; }
  __device__ __forceinline__ static Wide widen(Acc x) { return x; }
  __device__ __forceinline__ static Wide wcombine(Wide x, Wide y) { return x > y ? x : y; }
  __device__ __forceinline__ static Acc narrow(Wide x) { return x; }
  __device__ __forceinline__ static Vertex update(uint32_t, Acc acc, Vertex old_v, const Params&) {
    return acc > old_v ? acc : old_v;
  }
  __device__ __forceinline__ static bool better(Vertex cand, Vertex cur) { return cand > cur; }
  __device__ __forceinline__ static Vertex atomic_relax(Vertex* addr, Vertex cand) { return atomicMax(addr, cand); }
};

struct HopDistProgram {  // the reference's "SSSP" = BFS depth (sssp_gpu.cu:122: srcLabel + 1)
  using Vertex = uint32_t;
  using Acc = uint32_t;
  using Wide = uint32_t;
  struct Params { uint32_t unused; };
  static constexpr bool kNeedsOld = true;
  static constexpr bool kIsMax = false;
  static constexpr bool kWeighted = false;
  __device__ __forceinline__ static Acc identity() { return 0xFFFFFFFFu; }
  __device__ __forceinline__ static Acc gather(Vertex src_val) { return src_val + 1u; }  // INF = nv stays > nv
  __device__ __forceinline__ static Acc combine(Acc x, Acc y) { return x < y ? x : y; }
  __device__ __forceinline__ static Wide widen(Acc x) { return x; }
  __device__ __forceinline__ static Wide wcombine(Wide x, Wide y) { return x < y ? x : y; }
  __device__ __forceinline__ static Acc narrow(Wide x) { return x; }
  __device__ __forceinline__ static Vertex update(uint32_t, Acc acc, Vertex old_v, const Params&) {
    return acc < old_v ? acc : old_v;
  }
  __device__ __forceinline__ static bool better(Vertex cand, Vertex cur) { return cand < cur; }
  __device__ __forceinline__ static Vertex atomic_relax(Vertex* addr, Vertex cand) { return atomicMin(addr, cand); }
};

constexpr uint32_t kDistInf = 0xFFFFFFFFu;  // LUXB_DIST_INF

// D[u] + w without wrap-around: INF + w = INF, and a sum that would reach 2^32 - 1 reads as unreachable (w >= 0)
__host__ __device__ __forceinline__ uint32_t sat_add(uint32_t d, int32_t w) {
  const uint64_t s = (uint64_t)d + (uint32_t)w;
  return s < kDistInf ? (uint32_t)s : kDistInf;
}

// Weighted SSSP (no reference counterpart): D[v] = min(D[v], min over in-edges sat_add(D[u], w(u,v))), INF = 2^32 - 1.
// The weight enters per edge, so the kernels carry the source's raw label and call gather(label, w) where they read
// the edge's weight.
struct WeightedDistProgram {
  using Vertex = uint32_t;
  using Acc = uint32_t;
  using Wide = uint32_t;
  struct Params { uint32_t unused; };
  static constexpr bool kNeedsOld = true;
  static constexpr bool kIsMax = false;
  static constexpr bool kWeighted = true;
  __device__ __forceinline__ static Acc identity() { return kDistInf; }
  __device__ __forceinline__ static Acc gather(Vertex src_val, int32_t w) { return sat_add(src_val, w); }
  __device__ __forceinline__ static Acc combine(Acc x, Acc y) { return x < y ? x : y; }
  __device__ __forceinline__ static Wide widen(Acc x) { return x; }
  __device__ __forceinline__ static Wide wcombine(Wide x, Wide y) { return x < y ? x : y; }
  __device__ __forceinline__ static Acc narrow(Wide x) { return x; }
  __device__ __forceinline__ static Vertex update(uint32_t, Acc acc, Vertex old_v, const Params&) {
    return acc < old_v ? acc : old_v;
  }
  __device__ __forceinline__ static bool better(Vertex cand, Vertex cur) { return cand < cur; }
  __device__ __forceinline__ static Vertex atomic_relax(Vertex* addr, Vertex cand) { return atomicMin(addr, cand); }
};

}  // namespace luxb
