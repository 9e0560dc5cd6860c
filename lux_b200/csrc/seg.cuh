// seg.cuh — flagged segmented-scan sweep: the PageRank pull gather with ~4x fewer instructions per edge than the
// merge-path tiles of pull.cuh.  (Replaces pr_kernel, pagerank_gpu.cu:49-102.)
//
// Why.  In pull_tile_kernel the binary search, serial merge walk and per-vertex bookkeeping cost as many instructions as
// the gathers (about 2.2 warp instructions per merge item).  Once the hot gathers move to shared memory (panel.cuh) the
// instruction stream IS the bound.  This kernel drops the vertex-end markers altogether:
//   * the edge stream carries its own structure: the top bit of an edge word says "this edge starts a new destination
//     vertex" (head flag); the rest is the gather id (31 bits: hot-packed id; panel: 15-bit offset into the block's table);
//   * close_vtx[j] = the vertex whose in-edge list ENDS where head j begins (one u32 per non-empty vertex instead of
//     one row_end word per vertex; vertices without in-edges are handled by empties_kernel).  The group streams of the
//     split (panel, cold-hub; panel.cuh) close their slots in slot order, so they keep no such list: per piece t,
//     piece_slot[t] = (slot0, real range) and head k of the piece closes slot slot0 + k (kSlots);
//   * a warp owns a PIECE of kRounds x 32 x kV consecutive edges; per round each lane loads kV (8 or 16) consecutive words
//     with 128-bit shared-memory loads, issues its kV gathers, reduces them serially up to the head flags, and one
//     segmented warp-shuffle scan stitches the lanes; completed sums are staged in shared memory and written by a
//     lane-strided pass (update() + coalesced close_vtx loads, or consecutive slots).  The running carry across rounds is kept in the
//     program's wide type (fp64 for PageRank);
//   * the stream is padded with head-flagged dummy edges to whole stages, so the kernel has no bounds checks;
//   * pieces are claimed stage by stage from a global counter by a producer warp that streams the words with ONE TMA
//     bulk copy per stage (kWarps pieces, 8-32 KB) into a shared-memory ring (full/empty mbarriers) — same plumbing
//     as pull.cuh; a segment that spans pieces is finished by the same three fix-up kernels (head/tail partials).
// Deterministic: fixed reduction shape per piece, fix-up in ascending piece order.
// kPanel = true: 16-bit words, gathers from the shared-memory table of the current hot source block (panel.cuh).
#pragma once
#include "common.cuh"
#include "programs.cuh"
#include "pull.cuh"
#include "panel.cuh"

namespace luxb {

constexpr uint32_t kDummyVtx = 0xFFFFFFFFu;

template <int kWarps_, int kStages_, int kRounds_, bool kPanel_, int kTab_, int kV_ = 8>
struct SegShape {
  static constexpr int kWarps = kWarps_;
  static constexpr int kThreads = 32 * (kWarps + 1);
  static constexpr int kStages = kStages_;
  static constexpr int kRounds = kRounds_;
  static constexpr bool kPanel = kPanel_;
  static constexpr bool kSlots = kPanel_;                 // heads close compact slots (piece_slot), not close_vtx
  static constexpr int kTab = kTab_;                      // shared-memory table (values); 0 for the L1 sweep
  static constexpr int kV = kV_;                          // consecutive edges per lane and round (8 or 16)
  static constexpr int kRound = 32 * kV;                  // edges per warp round
  static constexpr int kPiece = kRounds * kRound;         // edges per warp piece
  static constexpr int kStageEdges = kWarps * kPiece;     // edges per stage (one TMA bulk copy)
  static constexpr int kWordBytes = kPanel ? 2 : 4;
  static constexpr int kStageBytes = kStageEdges * kWordBytes;
  static constexpr int kSumElems = kRound + 8;
  static constexpr int kHdrElems = kWarps + 4;            // stage id, table generation, tile_v[t0 .. t0 + kWarps]
  static constexpr size_t kSmemBytes = (size_t)kTab * 4 + (size_t)kStages * kStageBytes + (size_t)kWarps * kSumElems * 4 +
                                       (2 * kStages + 1) * 8 + (size_t)kStages * kHdrElems * 4 + 16;
  static_assert(!kPanel || (kTab > 0 && kTab <= 32768 && kTab % 4 == 0), "panel offsets are 15 bit");
  static_assert(kStageBytes % 16 == 0, "TMA bulk copies move multiples of 16 bytes");
  static_assert(kV == 8 || kV == 16, "a lane reads its words with 128-bit loads");
};

// a main (L1-gather) shape sweeping a group stream: the cold-hub stream
template <class Base>
struct SlotShape : Base {
  static constexpr bool kSlots = true;
};

template <class Prog>
struct SegArgs {
  PullArgs<Prog> p;          // out / update() parameters / hub_bits / raw_out / head+tail partials / tile_v / close_vtx
  const void* words;         // [n_stages * kStageEdges] flagged edge words (u32, or u16 for the panel)
  uint32_t n_stages;
  uint32_t* tile_counter;
  // panel only
  uint32_t bs, n_blocks;
  uint32_t super_end[kPanelMaxBlocks];
  // group streams (Shape::kSlots): [n_tiles] slot0 and real range of every piece, in place of p.close_vtx
  const uint2* piece_slot;
};

template <class Prog, class Shape>
__global__ void __launch_bounds__(Shape::kThreads, Shape::kPanel ? 1 : 2) seg_tile_kernel(const __grid_constant__ SegArgs<Prog> a) {
  using Acc = typename Prog::Acc;
  using Vertex = typename Prog::Vertex;
  using Wide = typename Prog::Wide;
  constexpr int kStages = Shape::kStages, kWarps = Shape::kWarps, kRounds = Shape::kRounds, kV = Shape::kV;
  constexpr bool kPanel = Shape::kPanel, kSlots = Shape::kSlots;
  static_assert(sizeof(Acc) == 4 && sizeof(Vertex) == 4, "4-byte vertex values");

  extern __shared__ __align__(128) unsigned char smem_raw[];
  Vertex* tab = reinterpret_cast<Vertex*>(smem_raw);                                   // kTab values (panel)
  unsigned char* w_buf = smem_raw + (size_t)Shape::kTab * 4;                             // kStages x kStageBytes
  Acc* sums_all = reinterpret_cast<Acc*>(w_buf + (size_t)kStages * Shape::kStageBytes);  // kWarps x kSumElems
  uint64_t* full = reinterpret_cast<uint64_t*>(sums_all + (size_t)kWarps * Shape::kSumElems);
  uint64_t* empty = full + kStages;
  uint64_t* tab_full = empty + kStages;
  uint32_t* hdr_all = reinterpret_cast<uint32_t*>(tab_full + 1);

  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;

  if (threadIdx.x == 0) {
    for (int s = 0; s < kStages; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], kWarps); }
    mbar_init(tab_full, 1);
    fence_mbar_init();
  }
  __syncthreads();

  if (warp == kWarps) {
    // ===== producer warp: claims stages from a global counter, keeps the right table resident (panel), streams words =====
    const uint64_t policy = l2_policy_evict_first();
    uint32_t cur_b = 0, gen = 0;
    bool loaded = false;
    for (uint32_t n = 0;; ++n) {
      const int s = n % kStages;
      if (n >= (uint32_t)kStages) mbar_wait(&empty[s], ((n / kStages) - 1) & 1u);
      uint32_t T = 0;
      if (lane == 0) T = atomicAdd(a.tile_counter, 1u);
      T = __shfl_sync(0xffffffffu, T, 0);
      uint32_t* hdr = hdr_all + s * Shape::kHdrElems;
      if (T >= a.n_stages) {
        if (lane == 0) { hdr[0] = 0xFFFFFFFFu; mbar_arrive(&full[s]); }
        break;
      }
      if (kPanel) {
        uint32_t b = cur_b;
        while (b + 1 < a.n_blocks && T >= a.super_end[b]) ++b;
        if (!loaded || b != cur_b) {
          // all consumers must be done with the stages issued so far (they gather from the old table)
          for (int q = 0; q < kStages; ++q) {
            if (n > (uint32_t)q) {
              const uint32_t m = n - 1 - ((n - 1 - q) % kStages);  // latest use of ring stage q
              mbar_wait(&empty[q], (m / kStages) & 1u);
            }
          }
          cur_b = b;
          loaded = true;
          ++gen;
          if (lane == 0) {
            const uint32_t bytes = a.bs * 4u;
            mbar_arrive_expect_tx(tab_full, bytes);
            const char* gsrc = reinterpret_cast<const char*>(a.p.x_hot + (size_t)b * a.bs);
            char* sdst = reinterpret_cast<char*>(tab);
            const uint64_t keep = l2_policy_evict_last();
            for (uint32_t off = 0; off < bytes; off += 32768u) {
              const uint32_t chunk = bytes - off < 32768u ? bytes - off : 32768u;
              bulk_g2s(sdst + off, gsrc + off, chunk, tab_full, keep);
            }
          }
          __syncwarp();
        }
      }
      const uint64_t t0 = (uint64_t)T * kWarps;
      if (lane <= kWarps) hdr[2 + lane] = __ldg(a.p.tile_v + t0 + lane);
      __syncwarp();
      if (lane == 0) {
        hdr[0] = T;
        hdr[1] = gen;
        mbar_arrive_expect_tx(&full[s], (uint32_t)Shape::kStageBytes);
        const char* gsrc = reinterpret_cast<const char*>(a.words) + (size_t)T * Shape::kStageBytes;
        char* sdst = reinterpret_cast<char*>(w_buf) + (size_t)s * Shape::kStageBytes;
        for (uint32_t off = 0; off < (uint32_t)Shape::kStageBytes; off += 32768u) {
          const uint32_t chunk = Shape::kStageBytes - off < 32768u ? Shape::kStageBytes - off : 32768u;
          bulk_g2s(sdst + off, gsrc + off, chunk, &full[s], policy);
        }
      }
      __syncwarp();
    }
    return;
  }

  // ===== consumer warps =====
  Acc* sums = sums_all + (size_t)warp * Shape::kSumElems;
  uint32_t my_gen = 0;
  const uint64_t pol_hot = a.p.l2_hints ? l2_policy_evict_last() : l2_policy_evict_normal();
  const uint64_t pol_cold = a.p.l2_hints ? l2_policy_evict_first() : l2_policy_evict_normal();
  for (uint32_t n = 0;; ++n) {
    const int s = n % kStages;
    mbar_wait(&full[s], (n / kStages) & 1u);
    const uint32_t* hdr = hdr_all + s * Shape::kHdrElems;
    const uint32_t T = hdr[0];
    if (T == 0xFFFFFFFFu) break;
    if (kPanel) {
      const uint32_t gen = hdr[1];
      if (gen != my_gen) { mbar_wait(tab_full, (gen - 1) & 1u); my_gen = gen; }
    }
    const uint32_t t = T * kWarps + warp;   // piece index
    const uint32_t jbase = hdr[2 + warp];   // heads before this piece
    const unsigned char* P = w_buf + (size_t)s * Shape::kStageBytes + (size_t)warp * Shape::kPiece * Shape::kWordBytes;
    uint32_t slot0 = 0, slot_end = 0;  // kSlots: head k (>= 1: head 0 is the fix-up's) closes slot slot0 + k if k < slot_end
    if constexpr (kSlots) {
      const uint2 ps = __ldg(a.piece_slot + t);
      slot0 = ps.x;
      slot_end = ps.y & ~kSlotLo;
    }

    Wide carry = Prog::widen(Prog::identity());  // warp-uniform: reduction of the edges since the last head
    bool seen = false;                           // a head has been met in this piece
    uint32_t n_closed = 0;                       // heads met so far in this piece

#pragma unroll 1
    for (int r = 0; r < kRounds; ++r) {
      // ---- kV consecutive edge words of this lane: 128-bit shared-memory loads ----
      uint32_t id[kV];
      uint32_t fm = 0;  // bit k: word k carries a head flag
      if (kPanel) {
        const uint4* src = reinterpret_cast<const uint4*>(P + ((size_t)r * Shape::kRound + lane * kV) * 2);
#pragma unroll
        for (int c = 0; c < kV / 8; ++c) {
          const uint4 q = src[c];
          const uint32_t w4[4] = {q.x, q.y, q.z, q.w};
#pragma unroll
          for (int k = 0; k < 4; ++k) {
            id[8 * c + 2 * k] = w4[k] & 0x7FFFu;
            id[8 * c + 2 * k + 1] = (w4[k] >> 16) & 0x7FFFu;
            fm |= ((w4[k] >> 15) & 1u) << (8 * c + 2 * k);
            fm |= (w4[k] >> 31) << (8 * c + 2 * k + 1);
          }
        }
      } else {
        const uint4* src = reinterpret_cast<const uint4*>(P + ((size_t)r * Shape::kRound + lane * kV) * 4);
#pragma unroll
        for (int c = 0; c < kV / 4; ++c) {
          const uint4 q = src[c];
          const uint32_t w4[4] = {q.x, q.y, q.z, q.w};
#pragma unroll
          for (int k = 0; k < 4; ++k) {
            id[4 * c + k] = w4[k] & 0x7FFFFFFFu;
            fm |= (w4[k] >> 31) << (4 * c + k);
          }
        }
      }
      // ---- gathers (compute()) ----
      Acc val[kV];
#pragma unroll
      for (int k = 0; k < kV; ++k) {
        if (kPanel) {
          val[k] = Prog::gather(tab[id[k]]);
        } else {
          const bool hot = id[k] < a.p.hot_n;
          const Vertex* ptr = hot ? a.p.x_hot + id[k] : a.p.x_old + (id[k] - a.p.hot_n);
          val[k] = Prog::gather(gather_load_l2(ptr, hot, pol_hot, pol_cold));
        }
      }
      if (r == kRounds - 1) {
        // the gathers above were issued with addresses computed from this stage's last words: every lane's reads of the
        // ring slot have completed, the slot can go back to the producer
        __syncwarp();
        if (lane == 0) mbar_arrive(&empty[s]);
      }
      // ---- where do this lane's completed sums go: exclusive prefix of the head counts ----
      const uint32_t cnt = __popc(fm);
      uint32_t incl = cnt;
#pragma unroll
      for (int off = 1; off < 32; off <<= 1) {
        const uint32_t up = __shfl_up_sync(0xffffffffu, incl, off);
        if (lane >= off) incl += up;
      }
      const uint32_t excl = incl - cnt;
      const uint32_t n_round = __shfl_sync(0xffffffffu, incl, 31);
      // the vertices this round completes: request their ids now, they are needed only after the reduction below
      constexpr int kPre = kSlots ? 1 : kV / 4;  // covers the typical number of completions per round (one per ~8 edges)
      uint32_t vpre[kPre];
      if constexpr (!kSlots) {
#pragma unroll
        for (int q = 0; q < kPre; ++q) {
          const uint32_t li = lane + 32 * q;
          vpre[q] = li < n_round ? __ldg(a.p.close_vtx + jbase + n_closed + li) : kDummyVtx;
        }
      }
      // ---- serial segmented reduction inside the lane ----
      Acc run = Prog::identity(), first_val = Prog::identity();
      uint32_t h = 0;  // heads met so far in this lane
      if (kPanel) {
        // shared-memory gathers: the instruction stream is the bound -> branch-free (selects + one predicated store per word)
#pragma unroll
        for (int k = 0; k < kV; ++k) {
          const bool f = (fm >> k) & 1u;
          const Acc closed = run;                               // what a head at word k completes
          if (f && h != 0) sums[excl + h] = closed;             // the lane's first completion waits for the scan below
          first_val = (f && h == 0) ? closed : first_val;
          run = f ? val[k] : Prog::combine(run, val[k]);
          h += f ? 1u : 0u;
        }
      } else {
        // L1 gathers: latency bound, heads are rare (1 in ~8 edges) -> skip the bookkeeping with a branch (measured faster)
#pragma unroll
        for (int k = 0; k < kV; ++k) {
          if ((fm >> k) & 1u) {
            if (h == 0) first_val = run; else sums[excl + h] = run;
            run = Prog::identity();
            ++h;
          }
          run = Prog::combine(run, val[k]);
        }
      }
      // ---- segmented inclusive scan of (has head, trailing partial) across the warp ----
      Acc sv = run;
      uint32_t sf = cnt ? 1u : 0u;
#pragma unroll
      for (int off = 1; off < 32; off <<= 1) {
        const Acc pv = __shfl_up_sync(0xffffffffu, sv, off);
        const uint32_t pf = __shfl_up_sync(0xffffffffu, sf, off);
        if (lane >= off) {
          if (!sf) sv = Prog::combine(pv, sv);
          sf |= pf;
        }
      }
      Acc ex_v = __shfl_up_sync(0xffffffffu, sv, 1);
      if (lane == 0) ex_v = Prog::identity();
      const Acc tail31 = __shfl_sync(0xffffffffu, sv, 31);
      const unsigned heads = __ballot_sync(0xffffffffu, cnt != 0);
      const bool defer_first = !seen;  // the piece's first head closes a vertex that may have begun in earlier pieces
      if (cnt) {
        const Acc value = Prog::combine(ex_v, first_val);
        if (lane == __ffs(heads) - 1) {  // first head of the round: the carry of the previous rounds belongs to it
          const Wide tot = Prog::wcombine(carry, Prog::widen(value));
          if (defer_first) a.p.head_partial[t] = Prog::narrow(tot); else sums[0] = Prog::narrow(tot);
        } else {
          sums[excl] = value;
        }
      }
      if (heads) { carry = Prog::widen(tail31); seen = true; } else { carry = Prog::wcombine(carry, Prog::widen(tail31)); }
      __syncwarp();
      // ---- update() + stores of the vertices completed in this round ----
      auto finish = [&](uint32_t li, uint32_t v) {
        if (li == 0 && defer_first) return;  // finished by the fix-up kernels (for piece 0 it is the dummy before head 0)
        if (v == kDummyVtx) return;
        if (kPanel) a.p.out[v] = sums[li];   // raw partial sum of a (block, hub) pair; combine_hub_kernel finishes the hub
        else store_vertex<Prog>(a.p, v, sums[li]);
      };
      if constexpr (kSlots) {
        for (uint32_t li = lane; li < n_round; li += 32) {
          const uint32_t k = n_closed + li;
          if (li == 0 && defer_first) continue;
          if (k >= slot_end) break;  // the rest are pads
          if (kPanel) a.p.out[slot0 + k] = sums[li];
          else store_vertex<Prog>(a.p, slot0 + k, sums[li]);
        }
      } else {
#pragma unroll
        for (int q = 0; q < kPre; ++q) {
          const uint32_t li = lane + 32 * q;
          if (li < n_round) finish(li, vpre[q]);
        }
        for (uint32_t li = lane + 32 * kPre; li < n_round; li += 32) finish(li, __ldg(a.p.close_vtx + jbase + n_closed + li));
      }
      n_closed += n_round;
      __syncwarp();
    }
    if (lane == 0) a.p.tail_partial[t] = Prog::narrow(carry);
  }
}

// ---- one-time construction of a flagged stream ---------------------------------------------------------------------
// one thread per "vertex" of a CSC (row_end inclusive): non-empty ones mark their first edge word and register
// themselves in the close list, if there is one (shifted by one: entry j+1 holds the vertex that owns head j).
struct StreamBlocks {            // vertices [vfirst[b], vfirst[b+1]) live in block b (main stream: one block)
  uint32_t n_blocks;
  uint32_t vfirst[kPanelMaxBlocks + 1];
  uint64_t ebase[kPanelMaxBlocks + 1];   // first edge (CSC index) of block b
  uint64_t wbase[kPanelMaxBlocks + 1];   // first stream word of block b
  uint64_t hshift[kPanelMaxBlocks + 1];  // pad heads inserted before block b
};

// the last block b < n with first[b] <= x (first[0] <= x; blocks may be empty)
template <class T>
__device__ __forceinline__ uint32_t find_block(const T* first, uint32_t n, uint64_t x) {
  uint32_t lo = 0, hi = n;  // first[lo] <= x, and first[hi] > x or hi == n
  while (hi - lo > 1) {
    const uint32_t mid = (lo + hi) >> 1;
    if ((uint64_t)first[mid] <= x) lo = mid; else hi = mid;
  }
  return lo;
}

__global__ void nonempty_flag_kernel(const uint64_t* __restrict__ row_end, uint32_t n_vtx, uint32_t* __restrict__ flag) {
  for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n_vtx; i += (uint64_t)gridDim.x * blockDim.x)
    flag[i] = row_end[i] > (i == 0 ? 0 : row_end[i - 1]) ? 1u : 0u;
}

template <class Word>
__global__ void stream_heads_kernel(const uint64_t* __restrict__ row_end, uint32_t n_vtx, const uint32_t* __restrict__ flag,
                                    const uint32_t* __restrict__ segrank, const __grid_constant__ StreamBlocks sb,
                                    Word* __restrict__ words, uint32_t* __restrict__ close_list) {
  constexpr Word kHead = (Word)1 << (sizeof(Word) * 8 - 1);
  for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n_vtx; i += (uint64_t)gridDim.x * blockDim.x) {
    if (!flag[i]) continue;
    const uint32_t b = find_block(sb.vfirst, sb.n_blocks, i);
    const uint64_t begin = i == 0 ? 0 : row_end[i - 1];
    words[begin - sb.ebase[b] + sb.wbase[b]] |= kHead;
    if (close_list) close_list[1 + (uint64_t)segrank[i] + sb.hshift[b]] = (uint32_t)i;
  }
}

// copy the ids of block-ordered edges into the stream (the ids must already be < 2^(bits-1))
template <class Word, class In>
__global__ void stream_copy_kernel(const In* __restrict__ ids, uint64_t e_cnt, const __grid_constant__ StreamBlocks sb,
                                   Word* __restrict__ words) {
  for (uint64_t e = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; e < e_cnt; e += (uint64_t)gridDim.x * blockDim.x) {
    const uint32_t b = find_block(sb.ebase, sb.n_blocks, e);
    words[e - sb.ebase[b] + sb.wbase[b]] = (Word)ids[e];
  }
}

// pad words [from, to) of the stream: head-flagged dummies (they close the block's last vertex, then dummy vertices)
template <class Word>
__global__ void stream_pad_kernel(Word* __restrict__ words, uint64_t from, uint64_t to) {
  constexpr Word kHead = (Word)1 << (sizeof(Word) * 8 - 1);
  for (uint64_t e = from + (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; e < to; e += (uint64_t)gridDim.x * blockDim.x) words[e] = kHead;
}

// heads per piece (exclusive scan of this = tile_v)
template <class Word>
__global__ void piece_heads_kernel(const Word* __restrict__ words, uint32_t n_pieces, uint32_t piece, uint32_t* __restrict__ cnt) {
  constexpr Word kHead = (Word)1 << (sizeof(Word) * 8 - 1);
  const unsigned lane = threadIdx.x & 31;
  const uint64_t warps_total = ((uint64_t)gridDim.x * blockDim.x) >> 5;
  for (uint64_t t = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; t < n_pieces; t += warps_total) {
    uint32_t c = 0;
    for (uint32_t k = lane; k < piece; k += 32) c += (words[t * piece + k] & kHead) ? 1u : 0u;
#pragma unroll
    for (int off = 16; off; off >>= 1) c += __shfl_xor_sync(0xffffffffu, c, off);
    if (lane == 0) cnt[t] = c;
  }
}

// compact slots of a group stream (its "vertices" are the (group, hub) pairs; non-empty ones are slots slot_base +
// segrank): piece t lies in one block b (blocks are padded to whole stages).  Block b's heads start at
// hb = segrank[vfirst[b]] + hshift[b]; head hb closes the previous block's last pad (a dummy), heads hb + 1 ..
// hb + n_b close the block's n_b slots in order, the heads after them close pads.  So head J of block b closes slot
// slot_base + J - 1 - hshift[b] when hb < J <= hb + n_b: piece t's real heads are one run.
__global__ void piece_slot_kernel(const uint32_t* __restrict__ tile_v, uint32_t n_pieces, uint32_t piece, const uint32_t* __restrict__ segrank,
                                  const __grid_constant__ StreamBlocks sb, uint32_t slot_base, uint2* __restrict__ piece_slot) {
  for (uint64_t t = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; t < n_pieces; t += (uint64_t)gridDim.x * blockDim.x) {
    const uint32_t b = find_block(sb.wbase, sb.n_blocks, t * piece);
    const int64_t r0 = segrank[sb.vfirst[b]], r1 = segrank[sb.vfirst[b + 1]];
    const int64_t hb = r0 + (int64_t)sb.hshift[b];
    const int64_t i0 = tile_v[t], i1 = tile_v[t + 1];
    const int64_t last = i1 < hb + 1 + (r1 - r0) ? i1 : hb + 1 + (r1 - r0);  // one past the piece's last real head
    const int64_t end = last > i0 ? last - i0 : 0;
    piece_slot[t] = make_uint2((uint32_t)((int64_t)slot_base + i0 - 1 - (int64_t)sb.hshift[b]), (uint32_t)end | (i0 == hb ? kSlotLo : 0u));
  }
}

// vertices without edges in the stream, split by the hub bitmap (order inside a list is irrelevant: warp-aggregated append)
__global__ void empty_split_kernel(const uint32_t* __restrict__ flag, uint32_t n_vtx, const uint32_t* __restrict__ hub_bits,
                                   uint32_t* __restrict__ plain, uint32_t* __restrict__ hubs, unsigned int* __restrict__ cursors) {
  const unsigned lane = threadIdx.x & 31;
  const uint64_t n_round = ((uint64_t)n_vtx + 31) & ~31ull;
  for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n_round; i += (uint64_t)gridDim.x * blockDim.x) {
    const bool e = i < n_vtx && !flag[i];
    const bool hub = e && hub_bits != nullptr && ((hub_bits[i >> 5] >> (i & 31)) & 1u);
    const unsigned mp = __ballot_sync(0xffffffffu, e && !hub), mh = __ballot_sync(0xffffffffu, hub);
    unsigned bp = 0, bh = 0;
    if (lane == 0) {
      if (mp) bp = atomicAdd(cursors + 0, (unsigned)__popc(mp));
      if (mh) bh = atomicAdd(cursors + 1, (unsigned)__popc(mh));
    }
    bp = __shfl_sync(0xffffffffu, bp, 0);
    bh = __shfl_sync(0xffffffffu, bh, 0);
    if (e && !hub) plain[bp + __popc(mp & ((1u << lane) - 1))] = (uint32_t)i;
    if (hub) hubs[bh + __popc(mh & ((1u << lane) - 1))] = (uint32_t)i;
  }
}

// vertices without in-edges in the swept stream get update(identity) — a constant when update() ignores the old value
// (PageRank): written once per value buffer; hubs among them get the raw identity EVERY iteration (combine_hub_kernel
// overwrites it with the final value)
template <class Prog>
__global__ void empties_kernel(const __grid_constant__ PullArgs<Prog> a, const uint32_t* __restrict__ empty_vtx, uint32_t n_empty) {
  for (uint64_t k = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; k < n_empty; k += (uint64_t)gridDim.x * blockDim.x)
    store_vertex<Prog>(a, empty_vtx[k], Prog::identity());
}

}  // namespace luxb
