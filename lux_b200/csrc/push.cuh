// push.cuh — frontier engine of the push model (CC / SSSP).  Replaces cc_push_kernel / sssp_push_kernel
// (components_gpu.cu:132-246), process_edge_dense/sparse (:48-82), bitmap_kernel (:248-281),
// convert_d2s_kernel (:283-315), the check kernels (:768-792, sssp_gpu.cu:773-798) and the label/frontier
// initialisation of push_init_task_impl (:733-739, sssp_gpu.cu:733-744).
//
// Frontier slot of partition p (FrontierHeader semantics, core/graph.h:100-106, push_model.inl:393-397):
//   header {u32 type, u32 numNodes}; DENSE_BITMAP: 1 bit per vertex, LSB-first, relative to row_left,
//   (R-L)/8+1 bytes; SPARSE_QUEUE: global vertex ids, capacity (R-L)/16 + 100.
// Our slot additionally carries, after the queue ids, the queue's new labels (same capacity) so that a sparse
// iteration exchanges (id, label) pairs instead of whole label slices.
#pragma once
#include "build.cuh"
#include "common.cuh"
#include "programs.cuh"

namespace luxb {

struct FrontierHeader {
  uint32_t type;
  uint32_t num_nodes;
};

// one entry per source partition, describing its frontier as exchanged after the previous iteration
struct FrontierDesc {
  const unsigned char* slot;  // header + payload
  uint32_t row_left;
  uint32_t n_part;
  uint32_t type;
  uint32_t count;  // queue entries (sparse) — dense uses n_part
};

struct PushArgs {
  FrontierDesc fr[LUXB_MAX_PARTS];
  int n_parts;
  const uint64_t* out_end;   // [nv] END offset of u's out-edge list inside this partition's CSR-by-source
  const uint32_t* out_dst;   // [ePart] destination ids (global), all inside [row_left, row_left + n_part)
  const uint32_t* lab;       // [nv] labels at iteration start (replica)
  uint32_t* cur;             // [n_part] this partition's working labels
  uint32_t row_left;
  // new frontier (sparse mode): exactly-once enqueue of changed destinations
  int new_sparse;
  uint32_t* new_count;       // &header.num_nodes of the new slot
  uint32_t* new_queue;
  uint32_t max_nodes;
  unsigned long long* edges_scanned;
  // sources with more than kPushBigDegree local out-edges are not relaxed inline: their edge list is cut into
  // kPushSegment-edge segments appended here and swept by push_big_kernel (one CTA per segment) — a hub with 10^6
  // out-edges would otherwise serialise on one CTA (the reference's kernel has exactly that problem)
  struct BigSeg { uint64_t begin; uint32_t len; uint32_t val; };
  BigSeg* big_list;
  uint32_t* big_count;
  uint32_t big_capacity;
  // weighted programs: [ePart] i32 weight of each out-edge, aligned with out_dst.  s_val / BigSeg::val then carry the
  // source's raw label and every edge adds its own weight
  const int32_t* out_w;
};

constexpr uint32_t kPushBigDegree = 2048;
constexpr uint32_t kPushSegment = 4096;

constexpr int kPushThreads = 256;

// one relaxation: atomics on this GPU's own slice only; returns true iff this thread must enqueue dst
template <class Prog>
__device__ __forceinline__ bool relax_edge(const PushArgs& a, uint32_t dstv, uint32_t cand) {
  uint32_t* addr = a.cur + (dstv - a.row_left);
  uint32_t seen = *reinterpret_cast<volatile uint32_t*>(addr);
  if (Prog::better(cand, seen)) {
    uint32_t prev = Prog::atomic_relax(addr, cand);
    // exactly-once enqueue: the thread that moves the label off its iteration-start value owns the append
    // (process_edge_sparse, components_gpu.cu:75-79)
    if (a.new_sparse && Prog::better(cand, prev) && prev == a.lab[dstv]) return true;
  }
  return false;
}
// warp-aggregated append to the new frontier queue: ONE atomic per warp
__device__ __forceinline__ void enqueue_warp(const PushArgs& a, bool enq, uint32_t dstv, int lane) {
  if (!a.new_sparse) return;
  unsigned m = __ballot_sync(0xffffffffu, enq);
  if (m) {
    int leader = __ffs(m) - 1;
    uint32_t pos = 0;
    if (lane == leader) pos = atomicAdd(a.new_count, (uint32_t)__popc(m));
    pos = __shfl_sync(0xffffffffu, pos, leader);
    if (enq) {
      pos += __popc(m & ((1u << lane) - 1));
      if (pos < a.max_nodes) a.new_queue[pos] = dstv;
    }
  }
}

// Each CTA takes kPushThreads frontier entries, scans their out-degrees (warp shuffles + smem), then all
// threads sweep the concatenated out-edge list; the owning source of an edge is found by binary search in the
// scanned offsets.  Relaxations are atomics on this GPU's own slice only (SURVEY fact 5); new frontier entries
// are appended with ONE atomic per warp (warp-aggregated).
template <class Prog>
__global__ void __launch_bounds__(kPushThreads) push_relax_kernel(const __grid_constant__ PushArgs a) {
  __shared__ uint64_t s_begin[kPushThreads];   // first out-edge of each entry's source
  __shared__ uint32_t s_scan[kPushThreads + 1];  // exclusive scan of degrees (clamped to u32 per CTA chunk)
  __shared__ uint32_t s_val[kPushThreads];     // relaxation value carried by the source
  __shared__ uint32_t s_warp[kPushThreads / 32];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;

  // flatten (partition, chunk) -> blockIdx.x
  uint32_t blk = blockIdx.x;
  int p = 0;
  uint32_t entries = 0;
  for (; p < a.n_parts; ++p) {
    entries = a.fr[p].type == LUXB_DENSE_BITMAP ? a.fr[p].n_part : a.fr[p].count;
    uint32_t nblk = (entries + kPushThreads - 1) / kPushThreads;
    if (blk < nblk) break;
    blk -= nblk;
  }
  if (p >= a.n_parts) return;
  const FrontierDesc& f = a.fr[p];
  uint32_t idx = blk * kPushThreads + tid;

  uint64_t deg = 0, begin = 0;
  uint32_t val = 0;
  if (idx < entries) {
    uint32_t u;
    bool active;
    if (f.type == LUXB_DENSE_BITMAP) {
      u = f.row_left + idx;
      const unsigned char* bitmap = f.slot + sizeof(FrontierHeader);
      active = (bitmap[idx >> 3] >> (idx & 7)) & 1;
    } else {
      const uint32_t* queue = reinterpret_cast<const uint32_t*>(f.slot + sizeof(FrontierHeader));
      u = queue[idx];
      active = true;
    }
    if (active) {
      uint64_t e1 = a.out_end[u];
      begin = u == 0 ? 0 : a.out_end[u - 1];
      deg = e1 - begin;
      if constexpr (Prog::kWeighted) val = a.lab[u];
      else val = Prog::gather(a.lab[u]);
      if (deg > kPushBigDegree) {
        uint32_t n_seg = (uint32_t)((deg + kPushSegment - 1) / kPushSegment);
        uint32_t pos = atomicAdd(a.big_count, n_seg);
        for (uint32_t q = 0; q < n_seg && pos + q < a.big_capacity; ++q) {
          PushArgs::BigSeg sg;
          sg.begin = begin + (uint64_t)q * kPushSegment;
          uint64_t rem = deg - (uint64_t)q * kPushSegment;
          sg.len = (uint32_t)(rem < kPushSegment ? rem : kPushSegment);
          sg.val = val;
          a.big_list[pos + q] = sg;
        }
        deg = 0;
      }
    }
  }
  // a single source with >= 2^32 local out-edges is impossible (e_part per CTA chunk is summed in u64 below)
  uint32_t d32 = (uint32_t)deg;
  uint32_t incl = d32;
#pragma unroll
  for (int off = 1; off < 32; off <<= 1) {
    uint32_t t = __shfl_up_sync(0xffffffffu, incl, off);
    if (lane >= off) incl += t;
  }
  if (lane == 31) s_warp[warp] = incl;
  __syncthreads();
  uint32_t wbase = 0;
  for (int w = 0; w < warp; ++w) wbase += s_warp[w];
  s_scan[tid] = wbase + incl - d32;
  s_begin[tid] = begin;
  s_val[tid] = val;
  if (tid == kPushThreads - 1) s_scan[kPushThreads] = wbase + incl;
  __syncthreads();
  const uint32_t total = s_scan[kPushThreads];
  if (tid == 0 && total) atomicAdd(a.edges_scanned, (unsigned long long)total);

  for (uint32_t base = 0; base < total; base += kPushThreads) {
    uint32_t e = base + tid;
    bool enq = false;
    uint32_t dstv = 0;
    if (e < total) {
      int lo = 0, hi = kPushThreads;  // last k with s_scan[k] <= e
      while (hi - lo > 1) {
        int mid = (lo + hi) >> 1;
        if (s_scan[mid] <= e) lo = mid; else hi = mid;
      }
      const uint64_t k = s_begin[lo] + (e - s_scan[lo]);
      dstv = a.out_dst[k];
      if constexpr (Prog::kWeighted) enq = relax_edge<Prog>(a, dstv, Prog::gather(s_val[lo], a.out_w[k]));
      else enq = relax_edge<Prog>(a, dstv, s_val[lo]);
    }
    enqueue_warp(a, enq, dstv, lane);
  }
}

// hubs: one CTA per kPushSegment-edge segment of a big source's out-edge list (persistent grid-stride)
template <class Prog>
__global__ void __launch_bounds__(kPushThreads) push_big_kernel(const __grid_constant__ PushArgs a) {
  const int lane = threadIdx.x & 31;
  uint32_t n = *a.big_count;
  if (n > a.big_capacity) n = a.big_capacity;
  for (uint32_t sidx = blockIdx.x; sidx < n; sidx += gridDim.x) {
    const PushArgs::BigSeg sg = a.big_list[sidx];
    if (threadIdx.x == 0) atomicAdd(a.edges_scanned, (unsigned long long)sg.len);
    for (uint32_t base = 0; base < sg.len; base += kPushThreads) {
      uint32_t e = base + threadIdx.x;
      bool enq = false;
      uint32_t dstv = 0;
      if (e < sg.len) {
        dstv = a.out_dst[sg.begin + e];
        if constexpr (Prog::kWeighted) enq = relax_edge<Prog>(a, dstv, Prog::gather(sg.val, a.out_w[sg.begin + e]));
        else enq = relax_edge<Prog>(a, dstv, sg.val);
      }
      enqueue_warp(a, enq, dstv, lane);
    }
  }
}

// frontier = {v : cur[v] != lab[v]} as a bitmap + count (bitmap_kernel, components_gpu.cu:248-281).
// One warp ballot produces one 32-bit bitmap word; count via popc, one atomic per CTA.
__global__ void frontier_diff_kernel(const uint32_t* __restrict__ lab_slice, const uint32_t* __restrict__ cur,
                                     uint32_t n_part, unsigned char* __restrict__ slot) {
  __shared__ uint32_t s_cnt;
  FrontierHeader* hdr = reinterpret_cast<FrontierHeader*>(slot);
  uint32_t* words = reinterpret_cast<uint32_t*>(slot + sizeof(FrontierHeader));
  if (threadIdx.x == 0) s_cnt = 0;
  __syncthreads();
  uint32_t local = 0;
  uint32_t n_round = (n_part + 31) & ~31u;
  for (uint64_t v = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; v < n_round; v += (uint64_t)gridDim.x * blockDim.x) {
    bool ch = v < n_part && lab_slice[v] != cur[v];
    unsigned m = __ballot_sync(0xffffffffu, ch);
    if ((threadIdx.x & 31) == 0) { words[v >> 5] = m; local += __popc(m); }
  }
  if (local) atomicAdd(&s_cnt, local);
  __syncthreads();
  if (threadIdx.x == 0 && s_cnt) atomicAdd(&hdr->num_nodes, s_cnt);
}

// bitmap -> queue of global ids (convert_d2s_kernel, components_gpu.cu:283-315), warp-aggregated append
__global__ void frontier_d2s_kernel(const unsigned char* __restrict__ dense_slot, uint32_t row_left, uint32_t n_part,
                                    unsigned char* __restrict__ sparse_slot, uint32_t max_nodes) {
  const uint32_t* words = reinterpret_cast<const uint32_t*>(dense_slot + sizeof(FrontierHeader));
  FrontierHeader* hdr = reinterpret_cast<FrontierHeader*>(sparse_slot);
  uint32_t* queue = reinterpret_cast<uint32_t*>(sparse_slot + sizeof(FrontierHeader));
  const unsigned lane = threadIdx.x & 31;
  uint32_t n_round = (n_part + 31) & ~31u;
  for (uint64_t v = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; v < n_round; v += (uint64_t)gridDim.x * blockDim.x) {
    unsigned m = words[v >> 5];  // same word for the whole warp
    if (m) {
      uint32_t base = 0;
      if (lane == 0) base = atomicAdd(&hdr->num_nodes, (uint32_t)__popc(m));
      base = __shfl_sync(0xffffffffu, base, 0);
      if ((m >> lane) & 1) {
        uint32_t pos = base + __popc(m & ((1u << lane) - 1));
        if (pos < max_nodes) queue[pos] = row_left + (uint32_t)v;
      }
    }
  }
}

// attach the queue entries' final labels (read after the relax kernel has finished)
__global__ void frontier_pack_labels_kernel(unsigned char* __restrict__ slot, uint32_t max_nodes, uint32_t row_left,
                                            const uint32_t* __restrict__ cur) {
  const FrontierHeader* hdr = reinterpret_cast<const FrontierHeader*>(slot);
  const uint32_t* queue = reinterpret_cast<const uint32_t*>(slot + sizeof(FrontierHeader));
  uint32_t* qlab = reinterpret_cast<uint32_t*>(slot + sizeof(FrontierHeader)) + max_nodes;
  uint32_t n = hdr->num_nodes < max_nodes ? hdr->num_nodes : max_nodes;
  for (uint32_t k = blockIdx.x * blockDim.x + threadIdx.x; k < n; k += gridDim.x * blockDim.x)
    qlab[k] = cur[queue[k] - row_left];
}

// receivers: scatter (id, label) pairs of a sparse slot into the label replica
__global__ void frontier_apply_kernel(const unsigned char* __restrict__ slot, uint32_t max_nodes, uint32_t count,
                                      uint32_t* __restrict__ lab) {
  const uint32_t* queue = reinterpret_cast<const uint32_t*>(slot + sizeof(FrontierHeader));
  const uint32_t* qlab = queue + max_nodes;
  for (uint32_t k = blockIdx.x * blockDim.x + threadIdx.x; k < count; k += gridDim.x * blockDim.x) lab[queue[k]] = qlab[k];
}

// ---- device-side frontier finalisation (components_gpu.cu:462-491 without host round trips) ------------------------
// The partition's new frontier exists as a bitmap candidate (slot D: built by frontier_diff_kernel) and / or a queue
// candidate (slot S: appended by the push kernels).  frontier_fix_kernel applies the reference's representation rules
// on the device — bitmap with fewer than max_nodes vertices -> demote to a queue (:469), queue that overflowed ->
// promote to a bitmap (:485) — the two conditional kernels run under device flags, frontier_final_kernel publishes the
// header, frontier_push_kernel ships slot + labels to every rank.  The host reads the P headers once per iteration.
struct FrontierCtl {
  uint32_t need_d2s;      // demote: rebuild the queue from the bitmap
  uint32_t need_promote;  // promote: rebuild the bitmap from the label diff
  uint32_t final_sparse;  // representation that is published
  uint32_t final_count;
};

__global__ void frontier_fix_kernel(unsigned char* slot_d, unsigned char* slot_s, uint32_t max_nodes, int dense_built, FrontierCtl* ctl) {
  if (blockIdx.x || threadIdx.x) return;
  FrontierHeader* hd = reinterpret_cast<FrontierHeader*>(slot_d);
  FrontierHeader* hs = reinterpret_cast<FrontierHeader*>(slot_s);
  ctl->need_d2s = 0;
  ctl->need_promote = 0;
  if (dense_built) {
    if (hd->num_nodes < max_nodes) { ctl->need_d2s = 1; hs->num_nodes = 0; }  // the queue is rebuilt from the bitmap
  } else if (hs->num_nodes >= max_nodes) {
    ctl->need_promote = 1;
    hd->num_nodes = 0;  // re-counted exactly by the diff (the reference over-counts here: defect B5)
  }
}

__global__ void frontier_final_kernel(unsigned char* slot_d, unsigned char* slot_s, int dense_built, FrontierCtl* ctl) {
  if (blockIdx.x || threadIdx.x) return;
  FrontierHeader* hd = reinterpret_cast<FrontierHeader*>(slot_d);
  FrontierHeader* hs = reinterpret_cast<FrontierHeader*>(slot_s);
  const bool sparse = dense_built ? ctl->need_d2s != 0 : ctl->need_promote == 0;
  ctl->final_sparse = sparse ? 1u : 0u;
  if (sparse) { hs->type = LUXB_SPARSE_QUEUE; ctl->final_count = hs->num_nodes; }
  else { hd->type = LUXB_DENSE_BITMAP; ctl->final_count = hd->num_nodes; }
}

// conditional variants: run only when *enable != 0 (the flags of FrontierCtl)
__global__ void frontier_diff_if_kernel(const uint32_t* __restrict__ enable, const uint32_t* __restrict__ lab_slice,
                                        const uint32_t* __restrict__ cur, uint32_t n_part, unsigned char* __restrict__ slot) {
  if (enable && *enable == 0) return;
  __shared__ uint32_t s_cnt;
  FrontierHeader* hdr = reinterpret_cast<FrontierHeader*>(slot);
  uint32_t* words = reinterpret_cast<uint32_t*>(slot + sizeof(FrontierHeader));
  if (threadIdx.x == 0) s_cnt = 0;
  __syncthreads();
  uint32_t local = 0;
  uint32_t n_round = (n_part + 31) & ~31u;
  for (uint64_t v = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; v < n_round; v += (uint64_t)gridDim.x * blockDim.x) {
    bool ch = v < n_part && lab_slice[v] != cur[v];
    unsigned m = __ballot_sync(0xffffffffu, ch);
    if ((threadIdx.x & 31) == 0) { words[v >> 5] = m; local += __popc(m); }
  }
  if (local) atomicAdd(&s_cnt, local);
  __syncthreads();
  if (threadIdx.x == 0 && s_cnt) atomicAdd(&hdr->num_nodes, s_cnt);
}

__global__ void frontier_d2s_if_kernel(const uint32_t* __restrict__ enable, const unsigned char* __restrict__ dense_slot, uint32_t row_left,
                                       uint32_t n_part, unsigned char* __restrict__ sparse_slot, uint32_t max_nodes) {
  if (*enable == 0) return;
  const uint32_t* words = reinterpret_cast<const uint32_t*>(dense_slot + sizeof(FrontierHeader));
  FrontierHeader* hdr = reinterpret_cast<FrontierHeader*>(sparse_slot);
  uint32_t* queue = reinterpret_cast<uint32_t*>(sparse_slot + sizeof(FrontierHeader));
  const unsigned lane = threadIdx.x & 31;
  uint32_t n_round = (n_part + 31) & ~31u;
  for (uint64_t v = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; v < n_round; v += (uint64_t)gridDim.x * blockDim.x) {
    unsigned m = words[v >> 5];
    if (m) {
      uint32_t base = 0;
      if (lane == 0) base = atomicAdd(&hdr->num_nodes, (uint32_t)__popc(m));
      base = __shfl_sync(0xffffffffu, base, 0);
      if ((m >> lane) & 1) {
        uint32_t pos = base + __popc(m & ((1u << lane) - 1));
        if (pos < max_nodes) queue[pos] = row_left + (uint32_t)v;
      }
    }
  }
}

__global__ void frontier_pack_labels_if_kernel(const uint32_t* __restrict__ enable, unsigned char* __restrict__ slot, uint32_t max_nodes,
                                               uint32_t row_left, const uint32_t* __restrict__ cur) {
  if (*enable == 0) return;
  const FrontierHeader* hdr = reinterpret_cast<const FrontierHeader*>(slot);
  const uint32_t* queue = reinterpret_cast<const uint32_t*>(slot + sizeof(FrontierHeader));
  uint32_t* qlab = reinterpret_cast<uint32_t*>(slot + sizeof(FrontierHeader)) + max_nodes;
  uint32_t n = hdr->num_nodes < max_nodes ? hdr->num_nodes : max_nodes;
  for (uint32_t k = blockIdx.x * blockDim.x + threadIdx.x; k < n; k += gridDim.x * blockDim.x) qlab[k] = cur[queue[k] - row_left];
}

// Frontier P2P push (SURVEY §8e): this partition's published slot — header + bitmap, or header + (id, label) pairs — and,
// for a bitmap, its label slice are stored straight into EVERY rank's slot table / label replica (peer pointers from
// cudaIpcOpenMemHandle; NVLink stores; disjoint ranges, no atomics across GPUs).  Sizes come from the device header.
struct FrontierPushArgs {
  const FrontierCtl* ctl;
  const unsigned char* slot_d;
  const unsigned char* slot_s;
  const uint32_t* cur;        // [n_part] this partition's labels
  uint32_t n_part, cap, row_left;
  int n_dst;
  unsigned char* dst_slot[LUXB_MAX_PARTS];  // this partition's slot inside every rank's slot table (own rank included)
  uint32_t* dst_lab[LUXB_MAX_PARTS];        // every rank's label replica
};
__global__ void frontier_push_kernel(const __grid_constant__ FrontierPushArgs a) {
  const bool sparse = a.ctl->final_sparse != 0;
  const uint32_t count = a.ctl->final_count;
  const uint32_t* src = reinterpret_cast<const uint32_t*>(sparse ? a.slot_s : a.slot_d);
  const uint64_t tid = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x, nth = (uint64_t)gridDim.x * blockDim.x;
  const uint32_t q = sparse ? (count < a.cap ? count : a.cap) : 0;
  const uint64_t words0 = 2 + (sparse ? (uint64_t)q : (count ? ((uint64_t)a.n_part + 31) / 32 : 0));
  for (int p = 0; p < a.n_dst; ++p) {
    uint32_t* d = reinterpret_cast<uint32_t*>(a.dst_slot[p]);
    for (uint64_t i = tid; i < words0; i += nth) d[i] = src[i];  // header + bitmap words / queue ids
    if (sparse) {
      const uint32_t* ql = src + 2 + a.cap;
      uint32_t* dl = d + 2 + a.cap;
      for (uint64_t i = tid; i < q; i += nth) dl[i] = ql[i];     // the queue entries' labels
    } else if (count) {
      uint32_t* dl = a.dst_lab[p] + a.row_left;
      for (uint64_t i = tid; i < a.n_part; i += nth) dl[i] = a.cur[i];  // label slice of a dense frontier
    }
  }
}

__global__ void frontier_headers_kernel(const unsigned char* __restrict__ fq_all, const __grid_constant__ PartTable pt,
                                        const uint64_t* __restrict__ slot_off, uint32_t* __restrict__ hdr_out) {
  const int p = threadIdx.x;
  if (p < pt.P) {
    const FrontierHeader* h = reinterpret_cast<const FrontierHeader*>(fq_all + slot_off[p]);
    hdr_out[2 * p] = h->type;
    hdr_out[2 * p + 1] = h->num_nodes;
  }
}

// CheckTask invariants over this partition's in-edges (A.6).  CC: label[dst] >= label[src];
// SSSP: label[src] != nv  =>  label[dst] <= label[src] + 1.
template <class Prog>
__global__ void check_kernel(const uint64_t* __restrict__ row_end_rel, const uint32_t* __restrict__ src, uint32_t n_part,
                             uint32_t row_left, uint32_t nv, const uint32_t* __restrict__ lab,
                             unsigned long long* __restrict__ mistakes) {
  unsigned long long bad = 0;
  for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n_part; i += (uint64_t)gridDim.x * blockDim.x) {
    uint64_t b = i == 0 ? 0 : row_end_rel[i - 1], e = row_end_rel[i];
    uint32_t ld = lab[row_left + i];
    for (uint64_t k = b; k < e; ++k) {
      uint32_t ls = lab[src[k]];
      if (Prog::kIsMax) bad += ld < ls; else bad += (ls != nv) && (ld > ls + 1);
    }
  }
  if (bad) atomicAdd(mistakes, bad);
}

// weighted SSSP: D[u] != INF  =>  D[v] <= sat_add(D[u], w(u,v)), over this partition's in-edges and their CSC weights
template <class Prog>
__global__ void check_kernel(const uint64_t* __restrict__ row_end_rel, const uint32_t* __restrict__ src, uint32_t n_part,
                             uint32_t row_left, const uint32_t* __restrict__ lab, unsigned long long* __restrict__ mistakes,
                             const int32_t* __restrict__ weight) {
  static_assert(Prog::kWeighted, "the weighted predicate");
  unsigned long long bad = 0;
  for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n_part; i += (uint64_t)gridDim.x * blockDim.x) {
    uint64_t b = i == 0 ? 0 : row_end_rel[i - 1], e = row_end_rel[i];
    uint32_t ld = lab[row_left + i];
    for (uint64_t k = b; k < e; ++k) {
      uint32_t ls = lab[src[k]];
      bad += (ls != kDistInf) && (ld > Prog::gather(ls, weight[k]));
    }
  }
  if (bad) atomicAdd(mistakes, bad);
}

}  // namespace luxb
