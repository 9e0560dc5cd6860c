// panel.cuh — source-blocked ("panel") half of the PageRank pull sweep: the split itself and the hub combine.
//
// Why (scripts/ubench_head.cu measures it): divergent 4-byte gathers through L1 run at one sector per cycle per SM —
// the wall the L1 sweep sits on; the same gathers from a table in SHARED memory run several times faster; distributed
// shared memory (ld.shared::cluster) is slower than L1; and a shared-memory table inside the L1-gather kernel starves
// L1 of the lines its misses need.  So the shared-memory gathers get a kernel launch of their own, in which NOTHING
// goes through L1:
//
//   * hub destinations  = local vertices with in-degree >= D (they own most edges of a skewed graph), ordered by
//     in-degree, descending (ties: ascending id);
//   * hot source blocks = the hot-packed value space [0, Ns) cut into NB blocks of BS <= 32768 values (BS * 4 B fits
//     shared memory next to the streaming ring);
//   * block b serves the hub prefix [0, N_b), N_b not increasing with b ("tiers"): tier 0 = the first blocks over all
//     hubs; later (less hot) blocks only over the hubs of highest in-degree, where a slot still collects enough edges;
//   * every edge (hot source of block b -> hub destination h < N_b) moves from the partition's CSC into the PANEL,
//     its in-edges stored as 15-BIT offsets into block b plus a head flag — 2 B of edge stream instead of 4 B.  Blocks
//     are padded to whole stages, so a stage never straddles two blocks.
//   * source GROUPS: group g < NB is panel block g, group NB + s is cold segment s (ColdSplit).  Group g serves the hub
//     prefix [0, N_g) (N_g = Nh for a segment); the group number is the edge's sort key.  A (group, hub) pair with at
//     least one edge is a SLOT.  Slots are numbered compactly and implicitly: groups ascending, hubs ascending inside a
//     group — the order in which the group streams close them — so a stream needs no close list (seg.cuh: slot0 +
//     head index per piece), and pairs without edges cost nothing.  The slot bitmap (one bit per (g, h < N_g), 32-hub
//     words, ceil(N_g / 32) words from SplitGroups::wbase[g]) and its per-word prefix of set bits give the combine the
//     slot of (g, h): pre[w] + popc(bits[w] & lanes below h).
// The panel stream is swept by seg_tile_kernel<kPanel> (seg.cuh): its producer warp keeps block b's values resident in
// shared memory (one TMA bulk load of BS * 4 B from the hot copies per block change) and its gathers are ld.shared.  It
// and the cold-hub stream write RAW partial sums into one array of slots.  The remaining edges stay in the "main"
// stream swept through L1; for hub vertices that sweep stores its raw sum too, and combine_hub_kernel adds main + the
// group partials in fp64 (fixed order: deterministic) and applies the vertex program's update().  Replaces pr_kernel
// (pagerank_gpu.cu:49-102).
#pragma once
#include "common.cuh"
#include "programs.cuh"
#include "pull.cuh"

namespace luxb {

// 177 blocks of 32768 values cover a 24 MB hot set; SegArgs / StreamBlocks carry per-block arrays as kernel parameters
constexpr int kPanelMaxBlocks = 256;
// 16-bit sort keys of the split: the edge's group (< kSplitKeyMain), main stream -> kSplitKeyMain
constexpr uint16_t kSplitKeyMain = 511;
constexpr int kSplitKeyBits = 9;

struct SplitGroups {
  uint32_t vbase[kSplitKeyMain + 1];  // Σ_{g' < g} N_g': N_g = vbase[g + 1] - vbase[g]; the dense (g, h) index vbase[g] + h
                                      // numbers the per-pair edge counts during construction
  uint32_t wbase[kSplitKeyMain + 1];  // first word of group g in the slot bitmap; [n_groups] = all words
};

// ---- one-time construction of the panel / main split --------------------------------------------------------------
__global__ void hub_flag_kernel(const uint64_t* __restrict__ row_end_rel, uint32_t n_part, uint32_t min_indeg,
                                uint32_t* __restrict__ flag) {
  for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n_part; i += (uint64_t)gridDim.x * blockDim.x) {
    uint64_t d = row_end_rel[i] - (i == 0 ? 0 : row_end_rel[i - 1]);
    flag[i] = d >= min_indeg ? 1u : 0u;
  }
}

// hub_idx = exclusive scan of flag.  Writes the hub list (local vertex ids, ascending; hub_order_key_kernel and a
// stable sort then order it by in-degree) and the bitmap the main kernel tests (bit v of word v / 32).
__global__ void hub_list_kernel(const uint32_t* __restrict__ flag, const uint32_t* __restrict__ hub_idx, uint32_t n_part,
                                uint32_t* __restrict__ hub_vtx, uint32_t* __restrict__ hub_bits) {
  const uint64_t n_round = ((uint64_t)n_part + 31) & ~31ull;
  for (uint64_t v = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; v < n_round; v += (uint64_t)gridDim.x * blockDim.x) {
    const bool f = v < n_part && flag[v];
    const unsigned m = __ballot_sync(0xffffffffu, f);
    if ((threadIdx.x & 31) == 0) hub_bits[v >> 5] = m;
    if (f) hub_vtx[hub_idx[v]] = (uint32_t)v;
  }
}

// sort key of hub h: its in-degree, descending (a stable ascending sort of ~indeg keeps ascending ids among ties)
__global__ void hub_order_key_kernel(const uint64_t* __restrict__ row_end_rel, const uint32_t* __restrict__ hub_vtx, uint32_t n_hub,
                                     uint32_t* __restrict__ key) {
  for (uint64_t h = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; h < n_hub; h += (uint64_t)gridDim.x * blockDim.x) {
    const uint32_t v = hub_vtx[h];
    key[h] = ~(uint32_t)(row_end_rel[v] - (v == 0 ? 0 : row_end_rel[v - 1]));
  }
}

// hub_idx[v] = position of hub v in the ordered hub list (entries of non-hubs are left as they are)
__global__ void hub_pos_kernel(const uint32_t* __restrict__ hub_vtx, uint32_t n_hub, uint32_t* __restrict__ hub_idx) {
  for (uint64_t h = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; h < n_hub; h += (uint64_t)gridDim.x * blockDim.x)
    hub_idx[hub_vtx[h]] = (uint32_t)h;
}

__global__ void edge_iota_kernel(uint64_t* __restrict__ payload, uint16_t* __restrict__ key, uint64_t n) {
  for (uint64_t e = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; e < n; e += (uint64_t)gridDim.x * blockDim.x) {
    payload[e] = e;
    key[e] = kSplitKeyMain;
  }
}

// Cold-hub split (PageRank on one rank, where the cold values are compacted right after the hot copies): edges from a
// COLD source (gather id >= H) into a hub move into a third flagged stream, ordered by cold source segment of `seg`
// values (group key0 + s).  Its kernel claims stages in order, so at any time all SMs gather from about one segment,
// which stays in L2 beside the persisting hot copies, instead of from the whole cold array at random.  Only hub
// destinations are split this way: their partials cost Nh * S slots, where splitting every destination would cost
// n_part * S.
struct ColdSplit {
  uint32_t hot_n;    // first cold gather id (H)
  uint32_t seg;      // cold values per segment; 0 = no cold-hub split
  uint32_t key0;     // sort key of segment 0 (= number of panel blocks)
};

// one warp per hub h (position in the ordered list): edges whose (hot-packed) source id lies below n_src, in a block b
// with h < n_pref[b], get key = b, payload = (h, e); with the cold split on, edges whose source is cold get key =
// cs.key0 + segment.  n_pref: [n_blocks] hub prefix of each block, n_blocks <= kPanelMaxBlocks.  cov_count[h]: the
// edges of hub h that left the main stream.
__global__ void hub_key_kernel(const uint64_t* __restrict__ row_end_rel, const uint32_t* __restrict__ src_gather,
                               const uint32_t* __restrict__ hub_vtx, uint32_t n_hub, uint32_t n_src, uint32_t bs,
                               const uint32_t* __restrict__ n_pref, uint32_t n_blocks,
                               uint16_t* __restrict__ key, uint64_t* __restrict__ payload, uint32_t* __restrict__ cov_count,
                               const ColdSplit cs) {
  __shared__ uint32_t s_pref[kPanelMaxBlocks];
  for (uint32_t i = threadIdx.x; i < n_blocks; i += blockDim.x) s_pref[i] = n_pref[i];
  __syncthreads();
  const unsigned lane = threadIdx.x & 31;
  const uint64_t warps_total = ((uint64_t)gridDim.x * blockDim.x) >> 5;
  for (uint64_t h = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; h < n_hub; h += warps_total) {
    const uint32_t v = hub_vtx[h];
    const uint64_t b = v == 0 ? 0 : row_end_rel[v - 1], e = row_end_rel[v];
    uint32_t cnt = 0;
    for (uint64_t k = b + lane; k < e; k += 32) {
      const uint32_t id = src_gather[k];
      if (id < n_src) {
        if (h < s_pref[id / bs]) {
          key[k] = (uint16_t)(id / bs);
          payload[k] = (h << 32) | k;
          ++cnt;
        }
      } else if (cs.seg != 0 && id >= cs.hot_n) {
        key[k] = (uint16_t)(cs.key0 + (id - cs.hot_n) / cs.seg);
        payload[k] = (h << 32) | k;
        ++cnt;
      }
    }
#pragma unroll
    for (int off = 16; off; off >>= 1) cnt += __shfl_xor_sync(0xffffffffu, cnt, off);
    if (lane == 0) cov_count[h] = cnt;
  }
}

__global__ void key_hist_kernel(const uint16_t* __restrict__ key, uint64_t n, unsigned long long* __restrict__ hist) {
  constexpr int kBins = kSplitKeyMain + 1;
  __shared__ unsigned int s_h[kBins];
  for (int i = threadIdx.x; i < kBins; i += blockDim.x) s_h[i] = 0;
  __syncthreads();
  // per-CTA counts stay below 2^32: each CTA sees at most n / gridDim.x + blockDim.x keys (n < 2^32 * gridDim.x)
  for (uint64_t e = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; e < n; e += (uint64_t)gridDim.x * blockDim.x)
    atomicAdd(&s_h[key[e]], 1u);
  __syncthreads();
  for (int i = threadIdx.x; i < kBins; i += blockDim.x)
    if (s_h[i]) atomicAdd(hist + i, (unsigned long long)s_h[i]);
}

// sorted (by group, stable) edges of groups starting at dense pair v0 -> their ids (gather id - group * bs: 16-bit block
// offsets for the panel, bs = 0 keeps the gather ids) + the edge count of every (group, hub) pair, counted from v0
template <class Word>
__global__ void group_fill_kernel(const uint16_t* __restrict__ key_sorted, const uint64_t* __restrict__ payload_sorted, uint64_t e_cnt,
                                  const uint32_t* __restrict__ src_gather, uint32_t bs, const __grid_constant__ SplitGroups sg,
                                  uint32_t v0, Word* __restrict__ ids, uint32_t* __restrict__ vcount) {
  for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < e_cnt; i += (uint64_t)gridDim.x * blockDim.x) {
    const uint32_t k = key_sorted[i];
    const uint64_t p = payload_sorted[i];
    const uint32_t e = (uint32_t)p, h = (uint32_t)(p >> 32);
    ids[i] = (Word)(src_gather[e] - k * bs);
    atomicAdd(vcount + (sg.vbase[k] - v0) + h, 1u);
  }
}

__global__ void main_fill_kernel(const uint64_t* __restrict__ payload_sorted, uint64_t e_main, const uint32_t* __restrict__ src_gather,
                                 uint32_t* __restrict__ main_src) {
  for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < e_main; i += (uint64_t)gridDim.x * blockDim.x)
    main_src[i] = src_gather[(uint32_t)payload_sorted[i]];
}

// in-degree of every local vertex inside the MAIN CSC = its in-degree minus the edges that moved to the other streams
__global__ void main_indeg_kernel(const uint64_t* __restrict__ row_end_rel, uint32_t n_part, const uint32_t* __restrict__ flag,
                                  const uint32_t* __restrict__ hub_idx, const uint32_t* __restrict__ cov_count,
                                  uint64_t* __restrict__ out) {
  for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n_part; i += (uint64_t)gridDim.x * blockDim.x) {
    uint64_t d = row_end_rel[i] - (i == 0 ? 0 : row_end_rel[i - 1]);
    if (flag[i]) d -= cov_count[hub_idx[i]];
    out[i] = d;
  }
}

// slot bitmap of groups [g0, g1) from the edge counts of their dense (group, hub) pairs (vcount, counted from pair v0):
// one warp per 32-hub word; bits past N_g stay clear
__global__ void slot_bits_kernel(const uint32_t* __restrict__ vcount, const __grid_constant__ SplitGroups sg, uint32_t g0, uint32_t g1,
                                 uint32_t v0, uint32_t* __restrict__ bits) {
  const unsigned lane = threadIdx.x & 31;
  const uint64_t warps_total = ((uint64_t)gridDim.x * blockDim.x) >> 5;
  for (uint64_t w = sg.wbase[g0] + (((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5); w < sg.wbase[g1]; w += warps_total) {
    uint32_t lo = g0, hi = g1;  // the group of word w: sg.wbase[lo] <= w < sg.wbase[hi]
    while (hi - lo > 1) {
      const uint32_t mid = (lo + hi) >> 1;
      if (sg.wbase[mid] <= w) lo = mid; else hi = mid;
    }
    const uint32_t h = (uint32_t)(w - sg.wbase[lo]) * 32u + lane;
    const bool f = h < sg.vbase[lo + 1] - sg.vbase[lo] && vcount[sg.vbase[lo] - v0 + h] != 0;
    const unsigned m = __ballot_sync(0xffffffffu, f);
    if (lane == 0) bits[w] = m;
  }
}

__global__ void popc_kernel(const uint32_t* __restrict__ bits, uint64_t n, uint32_t* __restrict__ out) {
  for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) out[i] = __popc(bits[i]);
}

// ---- per-iteration: hubs = main raw sum + panel partials (blocks b with h < N_b) + cold-segment partials, fp64, fixed
// order; then update() ---
template <class Prog>
struct CombineArgs {
  const uint32_t* hub_vtx;   // [n_hub] local vertex ids
  uint32_t n_hub, n_blocks, n_groups, row_left;
  SplitGroups sg;
  const uint32_t* slot_bits;  // [sg.wbase[n_groups]] bit h % 32 of word wbase[g] + h / 32: (g, h) has a slot
  const uint32_t* slot_pre;   // [sg.wbase[n_groups]] slots before the word (set bits of all earlier words)
  const typename Prog::Acc* partial;  // raw reductions, one per slot
  const typename Prog::Vertex* x_nat; // natural-order values of the previous iteration (update()'s old value)
  typename Prog::Vertex* out;  // [n_part] local; holds the main kernel's RAW sum for hub vertices on entry
  typename Prog::Params prm;
};

// A pair (g, h) without a slot has no edges: its partial would be the program's identity, which combines exactly (+0.0
// for PageRank's non-negative sums, the identity of max / min for labels), so skipping it changes no bit.
template <class Prog>
__global__ void combine_hub_kernel(const __grid_constant__ CombineArgs<Prog> a) {
  for (uint64_t h = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; h < a.n_hub; h += (uint64_t)gridDim.x * blockDim.x) {
    const uint32_t v = a.hub_vtx[h];
    typename Prog::Acc raw0;
    memcpy(&raw0, &a.out[v], sizeof(raw0));  // the main sweep left its RAW reduction in the value slot
    typename Prog::Wide t = Prog::widen(raw0);
    // h's bitmap word and lane: the same word for the 32 threads of a warp (the grid stride is a multiple of 32), so
    // the bitmap and prefix loads are broadcasts, and consecutive hubs with a slot sit at consecutive slots
    const uint32_t w = (uint32_t)(h >> 5), me = 1u << (h & 31), below = me - 1u;
    // block b serves h while h < N_b; N_b does not increase with b, so h < N_{b+7} means blocks b .. b+7 all do: their
    // loads are issued together, the adds keep block order.  Hubs are ordered by in-degree, so the threads of a warp
    // run about the same number of blocks.
    auto add8 = [&](uint32_t g) {  // groups g .. g + 7, which all serve h
      uint32_t bits[8], pre[8];
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        bits[i] = __ldg(a.slot_bits + a.sg.wbase[g + i] + w);
        pre[i] = __ldg(a.slot_pre + a.sg.wbase[g + i] + w);
      }
      typename Prog::Acc p[8];
#pragma unroll
      for (int i = 0; i < 8; ++i) p[i] = (bits[i] & me) ? a.partial[pre[i] + __popc(bits[i] & below)] : Prog::identity();
#pragma unroll
      for (int i = 0; i < 8; ++i)
        if (bits[i] & me) t = Prog::wcombine(t, Prog::widen(p[i]));
    };
    auto add = [&](uint32_t g) {
      const uint32_t bits = __ldg(a.slot_bits + a.sg.wbase[g] + w);
      if (bits & me) t = Prog::wcombine(t, Prog::widen(a.partial[__ldg(a.slot_pre + a.sg.wbase[g] + w) + __popc(bits & below)]));
    };
    uint32_t b = 0;
    for (; b + 8 <= a.n_blocks && h < a.sg.vbase[b + 8] - a.sg.vbase[b + 7]; b += 8) add8(b);
    for (; b < a.n_blocks && h < a.sg.vbase[b + 1] - a.sg.vbase[b]; ++b) add(b);
    uint32_t k = a.n_blocks;  // cold segments: every one serves all hubs
    for (; k + 8 <= a.n_groups; k += 8) add8(k);
    for (; k < a.n_groups; ++k) add(k);
    const typename Prog::Vertex oldv = Prog::kNeedsOld ? a.x_nat[a.row_left + v] : typename Prog::Vertex();
    const typename Prog::Vertex nv_ = Prog::update(a.row_left + v, Prog::narrow(t), oldv, a.prm);
    a.out[v] = nv_;
  }
}

}  // namespace luxb
