// pull.cuh — (1) the merge-path tile sweep over a partition's canonical CSC slice (replaces pr_kernel pagerank_gpu.cu:49-102
// and cc_pull_kernel / sssp_pull_kernel components_gpu.cu:85-130, sssp_gpu.cu:85-130): round 1's kernel, kept for graphs
// whose edge arrays stay in zero-copy host memory and as LUXB_SWEEP=merge; the default sweep is the flagged
// segmented-scan stream of seg.cuh.  (2) What both sweeps share: PullArgs, store_vertex (update() / raw sums for hub
// vertices), the gather loads with L1 / L2 policies, and the cross-tile FIX-UP (three kernels, or one chained scan).
//
// Merge-path design (not a translation).  The partition's work list is the MERGE of its nPart vertex-end markers
// (row_end) and its ePart in-edges (merge-path): cut into equal WARP TILES of W = 32 * kIPT merge items, so every
// warp gets the same amount of (vertex + edge) work no matter how skewed the in-degrees are.  Warps are completely
// independent — there is no __syncthreads in the hot loop — so the gather phase of one warp overlaps the reduction
// phase of the others and the load/store unit (the measured bottleneck: one 32-byte sector per cycle per SM for
// divergent 4-byte gathers) never idles.  Per warp tile:
//   1. a producer warp streams the row_end words and source ids of kWarps consecutive warp tiles (one "super-tile")
//      into a shared-memory ring with two TMA bulk copies (cp.async.bulk -> UBLKCP) behind a full/empty mbarrier
//      pair per stage — measured: ~1 small bulk copy per 400 cycles per SM, so one copy pair serves 8 warp tiles
//      (~7 KB) instead of one (per-warp copies made the kernel 2-4x slower).  L2 evict-first: streamed data must not displace the value array.  Consumer warps only
//      meet at these mbarriers and may drift kStages-1 super-tiles apart;
//      Weighted programs (weighted SSSP) add a third bulk copy per super-tile: the edge weights of the same range into
//      a weight ring next to the source-id ring;
//   2. every lane finds its merge-path start by binary search over <= W row_end words in shared memory, then issues
//      its (up to kIPT) gathers x[src] back to back on the read-only path — values land in REGISTERS in the order
//      the lane will consume them (no shared-memory round trip);
//   3. the lane walks its kIPT merge items serially: complete per-vertex reductions go to the warp's sums[] slot,
//      the leading and trailing partials are stitched across lanes by a segmented warp-shuffle scan (fixed shape ->
//      deterministic, unlike the reference's float atomicAdd);
//   4. a lane-strided pass applies the vertex program's update() and stores the new values coalesced.
// A vertex whose in-edge list crosses warp-tile boundaries is finished by the fix-up kernels below: a segmented scan
// over the tiles' tail partials (fp64 for PageRank) in ascending tile order, independent of the grid size.
#pragma once
#include "common.cuh"
#include "programs.cuh"

namespace luxb {

template <int kIPT_, int kWarps_, int kStages_>
struct PullShape {
  static constexpr int kIPT = kIPT_;            // merge items per lane
  static constexpr int kWarps = kWarps_;        // consumer warps per CTA (+1 producer warp)
  static constexpr int kThreads = 32 * (kWarps + 1);
  static constexpr int kTile = 32 * kIPT;       // merge items per warp tile
  static constexpr int kSuper = kTile * kWarps; // merge items per super-tile (one TMA pair)
  static constexpr int kStages = kStages_;      // ring depth
  static constexpr int kAElems = kSuper + 8;    // u32 low words of row_end (alignment slack + peek entry)
  static constexpr int kEElems = kSuper + 8;    // u32 source ids (alignment slack)
  static constexpr int kSumElems = kTile + 4;   // per consumer warp
  static constexpr int kHdrElems = kWarps + 4;  // per stage: super-tile id + tile_v[t0 .. t0 + kWarps]
  static constexpr size_t kSmemBytes = (size_t)kStages * (kAElems + kEElems) * 4 + (size_t)kWarps * kSumElems * 4 +
                                       2 * kStages * 8 + (size_t)kStages * kHdrElems * 4 + 16;
  static_assert(kIPT % 2 == 1, "kIPT must be odd: lane-contiguous smem reads are then bank-conflict free");
  static constexpr size_t kWRingOffset = (kSmemBytes + 15) & ~(size_t)15;  // weighted programs: weight ring after the rest
};

// dynamic shared memory of pull_tile_kernel<Prog, Shape>: weighted programs add a ring of kStages x kEElems weights
template <class Prog, class Shape>
constexpr size_t pull_smem_bytes() {
  return Prog::kWeighted ? Shape::kWRingOffset + (size_t)Shape::kStages * Shape::kEElems * 4 : Shape::kSmemBytes;
}

// weighted programs: [ePart + 8] i32 edge weights in CSC edge order (the same positions as src).  An empty base for the
// others, so that their PullArgs (and the SegArgs holding one) keep their layout byte for byte.
template <bool kWeighted>
struct PullWeights {};
template <>
struct PullWeights<true> {
  const int32_t* weight;
};

template <class Prog>
struct PullArgs : PullWeights<Prog::kWeighted> {
  const uint64_t* row_end;   // [nPart + 4] end offsets relative to the partition's first edge; padded with ~0
  const uint32_t* row_end32; // [nPart + 8] low 32 bits of row_end: what the tile kernel streams (differences inside
                             // a tile are < 2^32, so tile-relative offsets are exact modulo 2^32)
  const uint32_t* src;       // [ePart + 8] gather indices of the in-edges' sources (global ids, or hot-packed ids)
  const uint32_t* tile_v;    // [nTiles + 1] merge-path split: vertices consumed before each tile
  uint32_t n_part;           // vertices in this partition
  uint64_t e_part;           // edges in this partition
  uint32_t n_tiles;
  uint32_t row_left;         // global id of local vertex 0
  const typename Prog::Vertex* x_old;  // [nv] last iteration's values in natural (global id) order
  const typename Prog::Vertex* x_hot;  // [hot_n] contiguous copies of the hottest vertices' values (L2-persisting window)
  uint32_t hot_n;                      // ids < hot_n in `src` index x_hot, the others index x_old at (id - hot_n)
  const typename Prog::Vertex* x_nat;  // [nv] the same values in natural (global id) order, for update()'s old value
  typename Prog::Vertex* out;          // [nPart] this partition's new values (local index)
  typename Prog::Acc* head_partial;    // [nTiles] reduction of the tile's first completed vertex (tile-local part)
  typename Prog::Acc* tail_partial;    // [nTiles] reduction of the edges after the tile's last completed vertex
  typename Prog::Wide* carry;          // [nTiles] fix-up scratch: exclusive in-block carry
  uint32_t* carry_flag;                // [nTiles]
  typename Prog::Wide* block_agg;      // [nBlocks] fix-up scratch
  uint32_t* block_flag;                // [nBlocks]
  uint32_t* tile_counter;              // dynamic super-tile scheduler (zeroed before every launch)
  typename Prog::Params prm;
  // source-blocked sweep (panel.cuh): vertices whose bit is set in hub_bits get their RAW sum stored (no update(), no
  // peer stores) — combine_hub_kernel finishes them; raw_out != 0 does that for every vertex (the panel CSC's fix-up)
  const uint32_t* hub_bits;
  int raw_out;
  int l2_hints;  // gathers carry L2 eviction policies (hot: evict_last, cold: evict_first)
  // flagged segmented-scan sweep (seg.cuh): tile_v counts HEADS, and head j completes vertex close_vtx[j]
  const uint32_t* close_vtx;
};

// compact slots (panel.cuh): head k of piece t closes slot ps.x + k if lo <= k < end, ps.y = end | lo << 31.  lo = 1
// only for the first piece of a block, whose first head closes the previous block's last pad.
constexpr uint32_t kSlotLo = 0x80000000u;
__device__ __forceinline__ bool piece_slot_real(uint2 ps, uint32_t k) { return k >= (ps.y >> 31) && k < (ps.y & ~kSlotLo); }

template <class Prog>
__device__ __forceinline__ bool store_raw(const PullArgs<Prog>& a, uint32_t v) {
  if (a.raw_out) return true;
  return a.hub_bits != nullptr && ((__ldg(a.hub_bits + (v >> 5)) >> (v & 31)) & 1u);
}

template <class Prog>
__device__ __forceinline__ void store_vertex(const PullArgs<Prog>& a, uint32_t v, typename Prog::Acc sum) {
  using Vertex = typename Prog::Vertex;
  if (store_raw(a, v)) {
    Vertex r;
    static_assert(sizeof(Vertex) == sizeof(typename Prog::Acc), "raw sums travel in the value slot");
    memcpy(&r, &sum, sizeof(r));
    a.out[v] = r;
    return;
  }
  Vertex oldv = Prog::kNeedsOld ? __ldg(a.x_nat + a.row_left + v) : Vertex();
  Vertex nv_ = Prog::update(a.row_left + v, sum, oldv, a.prm);
  a.out[v] = nv_;
}

__global__ void tile_table_kernel(const uint64_t* __restrict__ row_end, uint32_t n_part, uint64_t e_part, uint32_t tile,
                                  uint32_t n_tiles, uint32_t* __restrict__ tile_v) {
  uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t > n_tiles) return;
  uint64_t total = (uint64_t)n_part + e_part;
  uint64_t d = (uint64_t)t * tile;
  if (d > total) d = total;
  uint64_t lo = d > e_part ? d - e_part : 0, hi = d < n_part ? d : n_part;
  while (lo < hi) {
    uint64_t mid = (lo + hi) >> 1;
    if (row_end[mid] <= d - 1 - mid) lo = mid + 1; else hi = mid;
  }
  tile_v[t] = (uint32_t)lo;
}

// Read-only gather with an L1 policy: hot copies are worth keeping in L1 (evict_last), a cold value is touched once
// per sweep and must not push them out (no_allocate).  LUXB_GATHER_HINTS=0 at compile time restores plain __ldg.
#ifndef LUXB_GATHER_HINTS
#define LUXB_GATHER_HINTS 1
#endif
template <class T>
__device__ __forceinline__ T gather_load(const T* p, bool hot) {
#if LUXB_GATHER_HINTS
  uint32_t v;
  if (hot) asm volatile("ld.global.nc.L1::evict_last.b32 %0, [%1];" : "=r"(v) : "l"(p));
  else asm volatile("ld.global.nc.L1::no_allocate.b32 %0, [%1];" : "=r"(v) : "l"(p));
  T r;
  memcpy(&r, &v, 4);
  return r;
#else
  (void)hot;
  return __ldg(p);
#endif
}

// the same with an L2 eviction policy per load (createpolicy): hot copies evict_last, cold values evict_first — the cold
// sectors (touched once per sweep) must not displace the hot lines in L2 either
template <class T>
__device__ __forceinline__ T gather_load_l2(const T* p, bool hot, uint64_t pol_hot, uint64_t pol_cold) {
  uint32_t v;
  if (hot) asm volatile("ld.global.nc.L1::evict_last.L2::cache_hint.b32 %0, [%1], %2;" : "=r"(v) : "l"(p), "l"(pol_hot));
  else asm volatile("ld.global.nc.L1::no_allocate.L2::cache_hint.b32 %0, [%1], %2;" : "=r"(v) : "l"(p), "l"(pol_cold));
  T r;
  memcpy(&r, &v, 4);
  return r;
}
__device__ __forceinline__ uint64_t l2_policy_evict_normal() {
  uint64_t pol;
  asm volatile("createpolicy.fractional.L2::evict_normal.b64 %0, 1.0;" : "=l"(pol));
  return pol;
}

__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}

template <class Prog, class Shape>
__global__ void __launch_bounds__(Shape::kThreads) pull_tile_kernel(const __grid_constant__ PullArgs<Prog> a) {
  using Acc = typename Prog::Acc;
  using Vertex = typename Prog::Vertex;
  static_assert(sizeof(Acc) == 4 && sizeof(Vertex) == 4, "4-byte vertex values");
  constexpr int kIPT = Shape::kIPT, kTile = Shape::kTile, kStages = Shape::kStages, kWarps = Shape::kWarps;

  extern __shared__ __align__(128) unsigned char smem_raw[];
  uint32_t* a_buf = reinterpret_cast<uint32_t*>(smem_raw);                       // kStages x kAElems
  uint32_t* e_buf = a_buf + (size_t)kStages * Shape::kAElems;                    // kStages x kEElems
  Acc* sums_all = reinterpret_cast<Acc*>(e_buf + (size_t)kStages * Shape::kEElems);  // kWarps x kSumElems
  uint64_t* full = reinterpret_cast<uint64_t*>(sums_all + (size_t)kWarps * Shape::kSumElems);
  uint64_t* empty = full + kStages;
  uint32_t* hdr_all = reinterpret_cast<uint32_t*>(empty + kStages);              // kStages x kHdrElems

  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const uint64_t total = (uint64_t)a.n_part + a.e_part;
  const uint32_t n_super = (a.n_tiles + kWarps - 1) / kWarps;

  if (threadIdx.x == 0) {
    for (int s = 0; s < kStages; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], kWarps); }
    fence_mbar_init();
  }
  __syncthreads();  // the only CTA-wide barrier: mbarrier initialisation

  if (warp == kWarps) {
    // ===== producer warp: claims super-tiles from a global counter (dynamic schedule keeps every CTA inside one
    // narrow window of the streamed arrays: few live DRAM pages / TLB entries, no tail imbalance), publishes the
    // tile geometry in the stage header and streams the slices with two TMA bulk copies =====
    const uint64_t policy = l2_policy_evict_first();
    for (uint32_t n = 0;; ++n) {
      const int s = n % kStages;
      if (n >= (uint32_t)kStages) mbar_wait(&empty[s], ((n / kStages) - 1) & 1u);
      uint32_t T = 0;
      if (lane == 0) T = atomicAdd(a.tile_counter, 1u);
      T = __shfl_sync(0xffffffffu, T, 0);
      uint32_t* hdr = hdr_all + s * Shape::kHdrElems;
      if (T >= n_super) {
        if (lane == 0) { hdr[0] = 0xFFFFFFFFu; mbar_arrive(&full[s]); }
        break;
      }
      const uint64_t t0 = (uint64_t)T * kWarps;
      if (lane <= kWarps) {
        uint64_t tt = t0 + lane < a.n_tiles ? t0 + lane : a.n_tiles;
        hdr[1 + lane] = __ldg(a.tile_v + tt);
      }
      __syncwarp();
      if (lane == 0) {
        hdr[0] = T;
        const uint64_t t1 = t0 + kWarps < a.n_tiles ? t0 + kWarps : a.n_tiles;
        const uint32_t i0 = hdr[1], i1 = hdr[1 + kWarps];
        const uint64_t d0 = t0 * kTile, d1 = t1 * kTile < total ? t1 * kTile : total;
        const uint64_t j0 = d0 - i0, j1 = d1 - i1;
        const uint32_t is = i0 & ~3u;
        const uint32_t bytes_a = ((i1 - is + 1) * 4 + 15) & ~15u;
        const uint64_t js = j0 & ~3ull;
        uint32_t bytes_e = (uint32_t)(((j1 - js) * 4 + 15) & ~15ull);
        if (j1 == j0) bytes_e = 0;
        if constexpr (Prog::kWeighted) {
          // third copy: the weights of the same edge range, into the weight ring
          mbar_arrive_expect_tx(&full[s], bytes_a + 2 * bytes_e);
          bulk_g2s(a_buf + (size_t)s * Shape::kAElems, a.row_end32 + is, bytes_a, &full[s], policy);
          if (bytes_e) {
            bulk_g2s(e_buf + (size_t)s * Shape::kEElems, a.src + js, bytes_e, &full[s], policy);
            int32_t* w_buf = reinterpret_cast<int32_t*>(smem_raw + Shape::kWRingOffset);
            bulk_g2s(w_buf + (size_t)s * Shape::kEElems, a.weight + js, bytes_e, &full[s], policy);
          }
        } else {
          mbar_arrive_expect_tx(&full[s], bytes_a + bytes_e);
          bulk_g2s(a_buf + (size_t)s * Shape::kAElems, a.row_end32 + is, bytes_a, &full[s], policy);
          if (bytes_e) bulk_g2s(e_buf + (size_t)s * Shape::kEElems, a.src + js, bytes_e, &full[s], policy);
        }
      }
      __syncwarp();
    }
    return;
  }

  // ===== consumer warps =====
  Acc* sums = sums_all + (size_t)warp * Shape::kSumElems;
  for (uint32_t n = 0;; ++n) {
    const int s = n % kStages;
    mbar_wait(&full[s], (n / kStages) & 1u);
    const uint32_t* hdr = hdr_all + s * Shape::kHdrElems;
    const uint32_t T = hdr[0];
    if (T == 0xFFFFFFFFu) break;
    const uint64_t t0 = (uint64_t)T * kWarps;
    const uint64_t t64 = t0 + warp;
    const bool active = t64 < a.n_tiles;
    const uint32_t t = (uint32_t)t64;
    const uint32_t si0 = hdr[1];
    const uint32_t i0 = hdr[1 + warp], i1 = hdr[2 + warp];
    const uint64_t sj0 = t0 * kTile - si0;
    const uint64_t d0 = (uint64_t)t * kTile, d1 = d0 + kTile < total ? d0 + kTile : total;
    const uint64_t j0 = d0 - i0, j1 = d1 - i1;
    const uint32_t n_v = i1 - i0, n_e = active ? (uint32_t)(j1 - j0) : 0u, n_items = n_v + n_e, j0lo = (uint32_t)j0;
    const uint32_t* A = a_buf + (size_t)s * Shape::kAElems + (si0 & 3u) + (i0 - si0);
    const uint32_t* E = e_buf + (size_t)s * Shape::kEElems + (uint32_t)(sj0 & 3ull) + (uint32_t)(j0 - sj0);

    if (active) {
      // ---- merge-path start of this lane: (i, j) with i + j = lane * kIPT ----
      uint32_t d = lane * kIPT;
      if (d > n_items) d = n_items;
      uint32_t lo = d > n_e ? d - n_e : 0, hi = d < n_v ? d : n_v;
      while (lo < hi) {
        uint32_t mid = (lo + hi) >> 1;
        if (A[mid] - j0lo <= d - 1 - mid) lo = mid + 1; else hi = mid;
      }
      uint32_t i = lo;
      const uint32_t j = d - lo;
      uint32_t i_next = __shfl_down_sync(0xffffffffu, i, 1);
      uint32_t j_next = __shfl_down_sync(0xffffffffu, j, 1);
      if (lane == 31) { i_next = n_v; j_next = n_e; }
      const uint32_t ne_lane = j_next - j;

      // ---- gather (compute()): up to kIPT independent read-only loads, parked in registers in walk order ----
      Acc val[kIPT];
#pragma unroll
      for (int k = 0; k < kIPT; ++k)
        if (k < (int)ne_lane) {
          const uint32_t id = E[j + k];
          const bool hot = id < a.hot_n;
          const Vertex* p = hot ? a.x_hot + id : a.x_old + (id - a.hot_n);
          if constexpr (Prog::kWeighted) {
            const int32_t* W = reinterpret_cast<const int32_t*>(smem_raw + Shape::kWRingOffset) + (size_t)s * Shape::kEElems +
                               (uint32_t)(sj0 & 3ull) + (uint32_t)(j0 - sj0);  // the weights at E's positions
            val[k] = Prog::gather(gather_load(p, hot), W[j + k]);
          } else {
            val[k] = Prog::gather(gather_load(p, hot));
          }
        }

      // ---- serial walk: edges [j, j_next) merged with vertex-end markers [i, i_next) ----
      Acc acc = Prog::identity();
      bool has_c = false;
      uint32_t first_i = 0;
      Acc first_val = Prog::identity();
      uint32_t aend = A[i] - j0lo;  // tile-relative end offset of vertex i (i == n_v reads a peek entry, never used)
#pragma unroll
      for (int k = 0; k < kIPT; ++k) {
        if (k < (int)ne_lane) {
          while (i < i_next && aend <= j + k) {  // vertex i has no more in-edges: its reduction is complete
            if (!has_c) { has_c = true; first_i = i; first_val = acc; } else { sums[i] = acc; }
            acc = Prog::identity();
            ++i;
            aend = A[i] - j0lo;
          }
          acc = Prog::combine(acc, val[k]);
        }
      }
      while (i < i_next) {  // markers after the lane's last edge
        if (!has_c) { has_c = true; first_i = i; first_val = acc; } else { sums[i] = acc; }
        acc = Prog::identity();
        ++i;
      }
      // ---- segmented inclusive scan of (has_c, trailing partial) across the warp ----
      Acc sv = acc;
      uint32_t sf = has_c ? 1u : 0u;
#pragma unroll
      for (int off = 1; off < 32; off <<= 1) {
        Acc pv = __shfl_up_sync(0xffffffffu, sv, off);
        uint32_t pf = __shfl_up_sync(0xffffffffu, sf, off);
        if (lane >= off) {
          if (!sf) sv = Prog::combine(pv, sv);
          sf |= pf;
        }
      }
      Acc ex_v = __shfl_up_sync(0xffffffffu, sv, 1);
      if (lane == 0) ex_v = Prog::identity();
      if (has_c) sums[first_i] = Prog::combine(ex_v, first_val);
      const Acc tail = __shfl_sync(0xffffffffu, sv, 31);
      __syncwarp();  // sums[] complete; every lane is done with this stage's A/E words
      if (lane == 0) {
        mbar_arrive(&empty[s]);  // release the ring slot to the producer
        a.tail_partial[t] = tail;
        if (n_v > 0) a.head_partial[t] = sums[0];
      }
      // ---- update() + coalesced stores (own replica and, in P2P mode, every peer's replica) ----
      for (uint32_t li = lane; li < n_v; li += 32) {
        if (li == 0 && t != 0) continue;  // may continue from previous tiles: finished by the fix-up kernels
        store_vertex<Prog>(a, i0 + li, sums[li]);
      }
      __syncwarp();  // sums[] reads done before the next tile's walk writes it
    } else {
      if (lane == 0) mbar_arrive(&empty[s]);
    }
  }
}

// ---- fix-up: vertices whose in-edge list spans several warp tiles ----------------------------------------------
// carry into tile t = combination, in ascending tile order, of the tail partials of the tiles since (and including)
// the last tile before t that completed a vertex.  A segmented scan in three small kernels:
//   1. per block of kFixBlock tiles: exclusive in-block scan -> carry[t], carry_flag[t]; block aggregate
//   2. one CTA scans the block aggregates (exclusive)
//   3. per tile that completes a vertex: total = carry (+ block prefix if no flagged tile precedes it in its block)
//      + head_partial[t]; update(); store.
constexpr int kFixBlock = 256;

template <class Prog>
__device__ __forceinline__ void seg_combine(uint32_t& f2, typename Prog::Wide& v2, uint32_t f1, typename Prog::Wide v1) {
  // (f1,v1) earlier, (f2,v2) later
  if (!f2) v2 = Prog::wcombine(v1, v2);
  f2 |= f1;
}

template <class Prog>
__global__ void __launch_bounds__(kFixBlock) pull_fixup_scan_kernel(const __grid_constant__ PullArgs<Prog> a) {
  using Wide = typename Prog::Wide;
  __shared__ Wide s_v[kFixBlock / 32];
  __shared__ uint32_t s_f[kFixBlock / 32];
  const uint32_t t = blockIdx.x * kFixBlock + threadIdx.x;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  uint32_t f = 0;
  Wide v = Prog::widen(Prog::identity());
  if (t < a.n_tiles) {
    f = a.tile_v[t + 1] > a.tile_v[t] ? 1u : 0u;
    v = Prog::widen(a.tail_partial[t]);
  }
  Wide sv = v;
  uint32_t sf = f;
#pragma unroll
  for (int off = 1; off < 32; off <<= 1) {
    Wide pv = __shfl_up_sync(0xffffffffu, sv, off);
    uint32_t pf = __shfl_up_sync(0xffffffffu, sf, off);
    if (lane >= off) seg_combine<Prog>(sf, sv, pf, pv);
  }
  if (lane == 31) { s_v[warp] = sv; s_f[warp] = sf; }
  __syncthreads();
  Wide wv = Prog::widen(Prog::identity());
  uint32_t wf = 0;
  for (int w = 0; w < warp; ++w) {  // (wf,wv) = aggregate of the preceding warps
    uint32_t f2 = s_f[w];
    Wide v2 = s_v[w];
    seg_combine<Prog>(f2, v2, wf, wv);
    wf = f2; wv = v2;
  }
  Wide ev = __shfl_up_sync(0xffffffffu, sv, 1);
  uint32_t ef = __shfl_up_sync(0xffffffffu, sf, 1);
  if (lane == 0) { ev = Prog::widen(Prog::identity()); ef = 0; }
  seg_combine<Prog>(ef, ev, wf, wv);
  if (t < a.n_tiles) { a.carry[t] = ev; a.carry_flag[t] = ef; }
  if (threadIdx.x == kFixBlock - 1) {
    uint32_t bf = sf;
    Wide bv = sv;
    seg_combine<Prog>(bf, bv, wf, wv);
    a.block_agg[blockIdx.x] = bv;
    a.block_flag[blockIdx.x] = bf;
  }
}

// exclusive scan of the block aggregates, in place, by one CTA: serial chunk per thread, then a segmented scan of the
// 1024 chunk aggregates with warp shuffles (two levels), then the chunk is rewritten as exclusive prefixes
template <class Prog>
__global__ void __launch_bounds__(1024) pull_fixup_blocks_kernel(const __grid_constant__ PullArgs<Prog> a, uint32_t n_blocks) {
  using Wide = typename Prog::Wide;
  __shared__ Wide s_v[32];
  __shared__ uint32_t s_f[32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const uint32_t per = (n_blocks + 1023) / 1024;
  const uint32_t b0 = threadIdx.x * per < n_blocks ? threadIdx.x * per : n_blocks;
  const uint32_t b1 = b0 + per < n_blocks ? b0 + per : n_blocks;
  Wide cv = Prog::widen(Prog::identity());
  uint32_t cf = 0;
  for (uint32_t b = b0; b < b1; ++b) {
    uint32_t f2 = a.block_flag[b];
    Wide v2 = a.block_agg[b];
    seg_combine<Prog>(f2, v2, cf, cv);
    cf = f2; cv = v2;
  }
  // inclusive segmented scan of (cf, cv) over the 1024 threads
  Wide sv = cv;
  uint32_t sf = cf;
#pragma unroll
  for (int off = 1; off < 32; off <<= 1) {
    Wide pv = __shfl_up_sync(0xffffffffu, sv, off);
    uint32_t pf = __shfl_up_sync(0xffffffffu, sf, off);
    if (lane >= off) seg_combine<Prog>(sf, sv, pf, pv);
  }
  if (lane == 31) { s_v[warp] = sv; s_f[warp] = sf; }
  __syncthreads();
  Wide wv = Prog::widen(Prog::identity());
  uint32_t wf = 0;
  for (int w = 0; w < warp; ++w) {
    uint32_t f2 = s_f[w];
    Wide v2 = s_v[w];
    seg_combine<Prog>(f2, v2, wf, wv);
    wf = f2; wv = v2;
  }
  Wide pv = __shfl_up_sync(0xffffffffu, sv, 1);  // exclusive prefix of this thread = agg(prev warps) (+) incl(lane-1)
  uint32_t pf = __shfl_up_sync(0xffffffffu, sf, 1);
  if (lane == 0) { pv = Prog::widen(Prog::identity()); pf = 0; }
  seg_combine<Prog>(pf, pv, wf, wv);
  for (uint32_t b = b0; b < b1; ++b) {  // rewrite aggregates as exclusive prefixes
    uint32_t f2 = a.block_flag[b];
    Wide v2 = a.block_agg[b];
    a.block_agg[b] = pv;
    a.block_flag[b] = pf;
    seg_combine<Prog>(f2, v2, pf, pv);
    pf = f2; pv = v2;
  }
}

template <class Prog>
__global__ void __launch_bounds__(kFixBlock) pull_fixup_apply_kernel(const __grid_constant__ PullArgs<Prog> a, const uint2* __restrict__ piece_slot) {
  using Wide = typename Prog::Wide;
  const uint32_t t = blockIdx.x * kFixBlock + threadIdx.x;
  if (t == 0 || t >= a.n_tiles) return;
  const uint32_t i0 = a.tile_v[t], i1 = a.tile_v[t + 1];
  if (i1 == i0) return;
  Wide c = a.carry[t];
  if (!a.carry_flag[t]) c = Prog::wcombine(a.block_agg[blockIdx.x], c);
  Wide totalw = Prog::wcombine(c, Prog::widen(a.head_partial[t]));
  uint32_t v = i0;
  if (piece_slot) {  // a group stream (seg.cuh): the piece's first head closes its first slot, or a pad
    const uint2 ps = piece_slot[t];
    if (!piece_slot_real(ps, 0)) return;
    v = ps.x;
  } else if (a.close_vtx) {
    v = a.close_vtx[i0];
    if (v == 0xFFFFFFFFu) return;  // a dummy (padding) vertex
  }
  store_vertex<Prog>(a, v, Prog::narrow(totalw));
}

// ---- the same fix-up in ONE launch: chained scan with decoupled look-back -----------------------------------------------
// Block b scans its kFixBlock tiles, publishes its aggregate, looks back over the predecessors' published aggregates /
// inclusive prefixes (the walk stops at the first aggregate that contains a completed vertex — almost always the
// immediate predecessor), publishes its own inclusive prefix and applies.  Publication = value word first, then a
// status word carrying the launch's epoch (no per-launch reset of the status array).  The combination follows tile
// order, but its fp64 association depends on which prefixes were already published, so the last bit of a carry may
// differ between runs (DESIGN §0); LUXB_FUSED_FIXUP=0 has a fixed association.
template <class Prog>
struct FixupChain {
  unsigned long long* value;   // [2 * n_blocks] aggregate / inclusive prefix values (Wide, bit-cast)
  unsigned long long* status;  // [2 * n_blocks] (epoch << 2) | (flag << 1) | 1  for aggregate (slot 2b) / prefix (2b + 1)
  unsigned long long* ticket;  // never reset: launch number `epoch` hands out tickets (epoch - 1) * n_blocks ...
  uint32_t epoch, n_blocks;
};

template <class Wide>
__device__ __forceinline__ unsigned long long wide_bits(Wide w) {
  unsigned long long u = 0;
  memcpy(&u, &w, sizeof(Wide));
  return u;
}
template <class Wide>
__device__ __forceinline__ Wide bits_wide(unsigned long long u) {
  Wide w;
  memcpy(&w, &u, sizeof(Wide));
  return w;
}

template <class Prog>
__global__ void __launch_bounds__(kFixBlock) pull_fixup_fused_kernel(const __grid_constant__ PullArgs<Prog> a, const FixupChain<Prog> ch,
                                                                  const uint2* __restrict__ piece_slot) {
  using Wide = typename Prog::Wide;
  __shared__ Wide s_v[kFixBlock / 32];
  __shared__ uint32_t s_f[kFixBlock / 32];
  __shared__ Wide s_pv;
  __shared__ uint32_t s_pf;
  __shared__ uint32_t s_b;
  // block index = order of arrival (a ticket), so a block only ever waits for blocks that are already running
  if (threadIdx.x == 0) s_b = (uint32_t)(atomicAdd(ch.ticket, 1ull) - (unsigned long long)(ch.epoch - 1) * ch.n_blocks);
  __syncthreads();
  const uint32_t b = s_b;
  const uint32_t t = b * kFixBlock + threadIdx.x;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  uint32_t f = 0;
  Wide v = Prog::widen(Prog::identity());
  uint32_t i0 = 0;
  if (t < a.n_tiles) {
    i0 = a.tile_v[t];
    f = a.tile_v[t + 1] > i0 ? 1u : 0u;
    v = Prog::widen(a.tail_partial[t]);
  }
  // in-block inclusive segmented scan
  Wide sv = v;
  uint32_t sf = f;
#pragma unroll
  for (int off = 1; off < 32; off <<= 1) {
    Wide pv = __shfl_up_sync(0xffffffffu, sv, off);
    uint32_t pf = __shfl_up_sync(0xffffffffu, sf, off);
    if (lane >= off) seg_combine<Prog>(sf, sv, pf, pv);
  }
  if (lane == 31) { s_v[warp] = sv; s_f[warp] = sf; }
  __syncthreads();
  Wide wv = Prog::widen(Prog::identity());
  uint32_t wf = 0;
  for (int w = 0; w < warp; ++w) {
    uint32_t f2 = s_f[w];
    Wide v2 = s_v[w];
    seg_combine<Prog>(f2, v2, wf, wv);
    wf = f2; wv = v2;
  }
  Wide ev = __shfl_up_sync(0xffffffffu, sv, 1);  // exclusive in-block prefix of this tile
  uint32_t ef = __shfl_up_sync(0xffffffffu, sf, 1);
  if (lane == 0) { ev = Prog::widen(Prog::identity()); ef = 0; }
  seg_combine<Prog>(ef, ev, wf, wv);
  if (threadIdx.x == kFixBlock - 1) {
    // block aggregate -> publish, look back, publish the inclusive prefix
    uint32_t af = sf;
    Wide av = sv;
    seg_combine<Prog>(af, av, wf, wv);
    const unsigned long long tag = (unsigned long long)ch.epoch << 2;
    volatile unsigned long long* st = ch.status;
    volatile unsigned long long* va = ch.value;
    va[2 * b] = wide_bits<Wide>(av);
    __threadfence();
    st[2 * b] = tag | (af << 1) | 1ull;
    uint32_t pf = 0;
    Wide pv = Prog::widen(Prog::identity());
    for (int64_t q = (int64_t)b - 1; q >= 0 && !pf; --q) {
      unsigned long long s_pre, s_agg;
      do {  // wait for the predecessor to publish something in this epoch
        s_pre = st[2 * q + 1];
        s_agg = st[2 * q];
      } while ((s_pre >> 2) != ch.epoch && (s_agg >> 2) != ch.epoch);
      __threadfence();
      const bool have_prefix = (s_pre >> 2) == ch.epoch;
      uint32_t qf = (uint32_t)(((have_prefix ? s_pre : s_agg) >> 1) & 1ull);
      Wide qv = bits_wide<Wide>(va[2 * q + (have_prefix ? 1 : 0)]);
      // (qf, qv) precedes (pf, pv)
      uint32_t nf = pf;
      Wide nv_ = pv;
      seg_combine<Prog>(nf, nv_, qf, qv);
      pf = nf; pv = nv_;
      if (have_prefix) break;
    }
    // inclusive prefix of this block = exclusive prefix (pf, pv) then aggregate (af, av)
    uint32_t inf = af;
    Wide inv = av;
    seg_combine<Prog>(inf, inv, pf, pv);
    va[2 * b + 1] = wide_bits<Wide>(inv);
    __threadfence();
    st[2 * b + 1] = tag | (inf << 1) | 1ull;
    s_pv = pv;
    s_pf = pf;
  }
  __syncthreads();
  if (t == 0 || t >= a.n_tiles || !f) return;
  // carry into this tile = block prefix then in-block exclusive prefix
  Wide c = ev;
  uint32_t cf = ef;
  seg_combine<Prog>(cf, c, s_pf, s_pv);
  const Wide totalw = Prog::wcombine(c, Prog::widen(a.head_partial[t]));
  uint32_t vtx = i0;
  if (piece_slot) {
    const uint2 ps = piece_slot[t];
    if (!piece_slot_real(ps, 0)) return;
    vtx = ps.x;
  } else if (a.close_vtx) {
    vtx = a.close_vtx[i0];
    if (vtx == 0xFFFFFFFFu) return;
  }
  store_vertex<Prog>(a, vtx, Prog::narrow(totalw));
}

}  // namespace luxb
