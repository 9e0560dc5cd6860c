// runtime.cuh — the per-rank host runtime state (replaces Graph + GraphPiece, core/graph.h:54-98, and the
// placement/ownership role of LuxMapper + Realm's FB allocator).  One luxb_graph = one rank = one GPU.
#pragma once
#include <vector>
#include "comm.h"
#include "common.cuh"
#include "panel.cuh"
#include "seg.cuh"
#include "push.cuh"
#include "bc.cuh"
#include "tc.cuh"
#include "kcore.cuh"
#include "truss.cuh"

// fix-up scratch of one tiled sweep (pull.cuh): per-tile partials and carries, per-block aggregates
struct FixupScratch {
  void* d_head = nullptr;
  void* d_tail = nullptr;
  void* d_carry = nullptr;
  uint32_t* d_carry_flag = nullptr;
  void* d_block_agg = nullptr;
  uint32_t* d_block_flag = nullptr;
  uint32_t n_fix_blocks = 0;
  unsigned long long* d_chain = nullptr;  // fused fix-up: [2 * n_fix_blocks] values then [2 * n_fix_blocks] status words
  uint32_t chain_epoch = 0;
};

// one CSC swept by a merge-path tile kernel, with its tile table and fix-up scratch
struct PullLayout {
  uint64_t* d_row_end = nullptr;    // [n_vtx + 4] (may be released once the tile table exists)
  uint32_t* d_row_end32 = nullptr;  // [n_vtx + 8]
  void* d_src = nullptr;            // u32 gather ids (main) or u16 block-local offsets (panel)
  uint32_t* d_tile_v = nullptr;
  uint32_t n_vtx = 0;
  uint64_t e_cnt = 0;
  uint32_t n_tiles = 0;
  FixupScratch fix;
  // flagged stream (seg.cuh): d_src holds the words, d_tile_v the heads before each piece, n_tiles the pieces
  uint32_t* d_close = nullptr;      // [1 + heads] vertex completed by each head (not for the group streams)
  uint2* d_piece_slot = nullptr;    // group streams: [n_tiles] compact slots closed by each piece (seg.cuh)
  uint32_t n_slots = 0;             // group streams: slots closed
  uint32_t* d_empty = nullptr;      // vertices without edges in this stream that are not hubs
  uint32_t n_empty = 0;
  uint32_t* d_empty_hub = nullptr;  // ... that are hubs (all their edges moved to the panel)
  uint32_t n_empty_hub = 0;
  uint32_t n_stages = 0;
  uint64_t n_words = 0;
};

// How the gather side and the pull sweeps are laid out (api.cu: build_hot_layout, build_panel_layout), read from the
// environment once at luxb_init (resolve_sweep_settings).  Modes: -1 (unset) automatic, 0 off, 1 forced.
struct SweepSettings {
  bool seg = true;             // LUXB_SWEEP=merge: the merge-path tiles of pull.cuh instead of the flagged streams
  int main_shape = 6, panel_shape = 1, cs_shape = 6;  // LUXB_SEG_MAIN_SHAPE, LUXB_SEG_PANEL_SHAPE, LUXB_CS_SHAPE (= main)
  int sb = -1;                 // LUXB_SB: the source-blocked split, automatic when the panel takes >= 1/5 of a large partition
  uint32_t sb_bs = 0;          // LUXB_SB_BS: values per hot source block (a multiple of 4, <= the panel table)
  uint32_t sb_blocks = 48;     // LUXB_SB_BLOCKS: tier 0, at most this many blocks over all hubs
  uint32_t sb_min_indeg = 64;  // LUXB_SB_MIN_INDEG: hub threshold
  // LUXB_SB_TIER: blocks past tier 0 over the rest of the hot set (automatic: where the cold-hub stream may be, on a
  // large partition), block b over the hubs of in-degree d with d * m_b >= LUXB_SB_SLOT_EDGES (expected edges per
  // slot; m_b = block b's share of the hubs' in-edges)
  int sb_tier = -1;
  double sb_slot_edges = 0.5;
  int cs = -1;                 // LUXB_CS: the cold-hub stream, automatic when its edges are >= kColdSplitMinShare
  double cs_seg_mb = 24.0;     // LUXB_CS_SEG_MB: its source segment (raised where the segments would not fit the keys)
  double hot_mb = 24.0;        // LUXB_HOT_MB: the hot set
  bool l2_persist = true;      // LUXB_L2_PERSIST=0: no persisting L2 window
  double l2_window_mb = -1.0;  // LUXB_L2_WINDOW_MB: cap on that window (< 0: unset)
  // LUXB_PANEL_SMS: one rank with the split: the panel kernel runs on this many SMs while the cold-hub and main
  // kernels run beside it on the others (api.cu: sweep_seg); 0, or >= the SM count: one after another
  int panel_sms = 40;
};

// dev aid: LUXB_PHASE_TIMING=1 prints the mean device time of each phase of a PageRank iteration at luxb_close.
// ev / tag: marks on the compute stream, each timing the phase since the previous mark; span_ev / spans: phases
// between two events of any stream (the concurrent sweep's side stream, its overlapped region)
struct PhaseTimer {
  struct Span { int begin, end, tag; };
  bool on = false, per_call = false;
  std::vector<cudaEvent_t> ev;
  std::vector<int> tag;
  std::vector<cudaEvent_t> span_ev;
  std::vector<Span> spans;
  double sum[15] = {0};
  double chain = 0;  // the compute stream's marks summed: the device time of the iterations
  long cnt = 0;
};

// col_filter (cf.cuh): the chunk table of this rank's destinations
struct CfState {
  uint32_t* chunk_first = nullptr;
  uint32_t* chunk_vtx = nullptr;
  uint32_t n_chunks = 0;
  float* partial = nullptr;
};

// betweenness centrality (bc.cuh): the BFS of the label engine, then per source the level lists, σ and δ; scores summed
// over sources
struct BcState {
  double* sigma = nullptr;       // [nv] path counts of the last source
  double* delta = nullptr;       // [nv] dependencies of the last source
  double* scores = nullptr;      // [nv] Σ δ over the sources processed (the handle's values)
  uint32_t* order = nullptr;     // [nv] reached ids sorted stably by level (weighted: by distance)
  double* lvl = nullptr;         // one level's sums, in level order (grown to the largest level seen)
  uint64_t lvl_cap = 0;
  uint32_t* off = nullptr;       // level_off[L + 1] (weighted: class_off, one entry per distinct distance)
  uint64_t off_cap = 0;
  uint32_t* split = nullptr;     // nranks > 1: [L][P + 1] every partition's piece of every level
  uint64_t split_cap = 0;
  void* sort_tmp = nullptr;
  size_t sort_bytes = 0;
  uint32_t* ctl = nullptr;       // [0..1] BcCtl of the level being summed, [2] deepest level (weighted: largest
                                 // distance), [3] weighted: reached vertices, [4] weighted: class count
  luxb::BcHub* hubs = nullptr;
  double* partial = nullptr;
  std::vector<uint32_t> h_off, h_split;  // host copies of this source's level_off / split
  bool has_source = false;
};

// triangle counting (tc.cuh): the oriented adjacency of the whole graph and the bins of this rank's range
struct TcState {
  uint64_t m = 0;                  // undirected simple edges
  uint64_t* off = nullptr;         // [nv + 1] out-list offsets
  uint32_t* dst = nullptr;         // [m] out-lists N+(u), ascending ids
  uint32_t* staged = nullptr;      // vertices of the grouped kernel
  uint64_t* stage_pre = nullptr;
  uint32_t* group = nullptr;
  uint32_t* big = nullptr;         // vertices of the big kernel
  uint32_t n_group = 0, n_big = 0;
  unsigned long long* t = nullptr;      // [nv] per-vertex counts (the handle's values)
  unsigned long long* total = nullptr;  // [1] sum of t
  unsigned int* next = nullptr;         // [2] work counters
  void* sum_tmp = nullptr;
  size_t sum_bytes = 0;
  int group_grid = 0, big_grid = 0;
};

// k-core decomposition (kcore.cuh): this rank's adjacency over all sources, the peel's state
struct KcoreState {
  uint64_t m = 0;                  // undirected simple edges (2 m adjacency entries over all ranks)
  uint64_t* off = nullptr;         // [nv + 1] offsets of every source's list of this rank's neighbours
  uint32_t* adj = nullptr;         // this rank's adjacency entries, targets in [row_left, row_right]
  uint32_t* deg0 = nullptr;        // [n_part] degrees
  uint32_t* deg = nullptr;         // [n_part] degrees during a run; check counters [2 n_part] after it
  uint32_t* core = nullptr;        // [nv] core numbers (the handle's values)
  uint32_t* alive[2] = {nullptr, nullptr};  // [n_part] alive lists
  uint32_t* piece[2] = {nullptr, nullptr};  // [n_part] this rank's pieces of F
  uint32_t* f = nullptr;           // [nv] the global F (several ranks)
  uint64_t* pre = nullptr;         // [nv + 1] slot offsets of F's lists
  luxb::KcoreRec* rec = nullptr;   // [1 + LUXB_MAX_PARTS] this rank's record, then every rank's
  luxb::KcoreRec* h_rec = nullptr; // pinned host copy of the gathered records
  unsigned long long* bad = nullptr;
  void* scan_tmp = nullptr;
  size_t scan_bytes = 0;
  int grid = 0;                    // resident CTAs of the scatter and the tally
};

// k-truss decomposition (truss.cuh): the edge table, TC's oriented lists with their edge ids, the symmetric adjacency,
// the peel's state.  Every rank holds all of it; a rank owns the edges [e_lo, e_hi) whose lo is in its range.
struct TrussState {
  uint64_t m = 0;                  // undirected simple edges
  uint32_t e_lo = 0, e_hi = 0;
  uint64_t* ekey = nullptr;        // [m] lo << 32 | hi, ascending: the edge ids
  TcState o;                       // oriented out-lists and this rank's bins (tc_orient_bins); o.next: work counters
  uint32_t* oid = nullptr;         // [m] edge id of every oriented position
  uint64_t* off = nullptr;         // [nv + 1] symmetric adjacency offsets
  uint64_t* adj = nullptr;         // [2m] neighbour << 32 | edge id, neighbours ascending inside each list
  uint32_t* sup0 = nullptr;        // [m] support of the input graph
  uint32_t* sup = nullptr;         // [m] support during a run (this rank's edges current)
  uint32_t* truss = nullptr;       // [m] τ
  uint8_t* st = nullptr;           // [m] alive / dying / dead
  uint32_t* tv = nullptr;          // [nv] max τ at every vertex (the handle's values)
  uint32_t* alive[2] = {nullptr, nullptr};  // [e_hi - e_lo] alive lists of this rank's edges
  uint32_t* piece[2] = {nullptr, nullptr};  // this rank's pieces of F
  uint32_t* f = nullptr;           // [m] the global F (several ranks)
  uint64_t* pre = nullptr;         // [m + 1] slot offsets of F's walks
  luxb::KcoreRec* rec = nullptr;   // [1 + LUXB_MAX_PARTS] this rank's record, then every rank's
  luxb::KcoreRec* h_rec = nullptr; // pinned host copy of the gathered records
  unsigned long long* bad = nullptr;
  void* scan_tmp = nullptr;
  size_t scan_bytes = 0;
  int grid = 0;                    // resident CTAs of the walk and the tally
  int group_grid = 0, big_grid = 0;
};

// one buffer the graph keeps: device memory, pinned host memory, or pinned host memory mapped into the device's
// address space
enum class MemKind : uint8_t { kDevice, kPinned, kMapped };
struct OwnedBuf { void* p; MemKind kind; };

struct luxb_graph {
  luxb_config cfg{};
  uint32_t nv = 0;
  uint64_t ne = 0;
  int P = 1;
  int parts_found = 0;  // partitions the reference's greedy scan produced (== P when the reference would accept)
  bool weighted = false;

  // global partition table (Graph::rowLeft/rowRight, core/graph.h:62)
  // the reference's split as reported by luxb_partition_bounds; rl / np / cl below are the WORK split in use (the same
  // unless cfg.balanced_split)
  uint32_t ref_rl[LUXB_MAX_PARTS]{};
  uint32_t ref_np[LUXB_MAX_PARTS]{};
  uint64_t ref_cl[LUXB_MAX_PARTS]{};
  uint32_t rl[LUXB_MAX_PARTS]{};
  uint32_t np[LUXB_MAX_PARTS]{};
  uint64_t cl[LUXB_MAX_PARTS]{};
  uint32_t cap[LUXB_MAX_PARTS]{};      // frontier queue capacity per partition (push_model.inl:393)
  uint64_t slot_off[LUXB_MAX_PARTS]{}; // our slot offsets inside fq buffers
  uint64_t slot_bytes[LUXB_MAX_PARTS]{};
  uint64_t fq_total = 0;

  // this rank's slice
  uint32_t row_left = 0, n_part = 0;
  uint64_t col_left = 0, e_part = 0;
  uint64_t* d_row_end = nullptr;  // [n_part + 4] relative end offsets + sentinels
  uint32_t* d_src = nullptr;      // [e_part + 8]
  int32_t* d_weight = nullptr;    // [e_part + 8] (col_filter)
  // the slice as swept by the merge-path kernel (pull.cuh): tile table, u32 row ends, fix-up scratch.  It borrows
  // d_row_end from the graph and leaves d_src unset: each sweep passes the gather ids it uses.
  PullLayout base;
  int pull_shape = 0;             // merge-path shape (LUXB_PULL_SHAPE), chosen by finish_layout

  cudaStream_t stream = nullptr;
  cudaEvent_t ev_begin = nullptr, ev_end = nullptr;
  int num_sms = 0;

  // app state
  bool inited = false;
  uint32_t* d_deg = nullptr;   // PageRank: global out-degrees
  void* d_val[2] = {nullptr, nullptr};  // replicas of the vertex values (labels: only [0])
  int cur = 0;
  // hot-packed gather layout (PageRank): hot copies live in d_hot, natural-order values in d_val[0/1]
  uint32_t hot_n = 0;
  void* d_hot = nullptr;             // [hot_n] hot copies (single buffer: refreshed in place after every iteration)
  uint32_t hot_off[LUXB_MAX_PARTS + 1]{};  // hot slots owned by partition p: [hot_off[p], hot_off[p+1])
  uint32_t* d_hot_order = nullptr;   // [hot_n (+ cold_n if cold_z)] vertex id held by each hot slot (descending out-degree)
  uint32_t* d_src_gather = nullptr;  // [e_part + 8] source ids rewritten as indices into Z
  // packed exchange (PageRank, nranks > 1): transfer arrays XT[2] = [hot by owner (hot_n) | cold-active by id (cold_n)]
  bool packed = false;
  uint32_t cold_n = 0;                       // vertices with 0 < out-degree < tau (all partitions)
  uint32_t cold_off[LUXB_MAX_PARTS + 1]{};   // cold-active vertices owned by partition p: [cold_off[p], cold_off[p+1])
  uint32_t* d_zperm = nullptr;               // [hot_n] global hot rank of the k-th entry of XT's hot part
  uint32_t* d_pack_list = nullptr;           // local indices of this rank's [hot | cold-active] vertices in transfer order
  float* d_xt[2] = {nullptr, nullptr};
  int cur_xt = 0;
  uint64_t xt_hot_chunk = 0, xt_cold_chunk = 0;  // equal chunks (elements) of the two balanced all-gathers; XT = [P hot chunks | P cold chunks]
  // the cold part of the exchange runs on a second stream, overlapped with the next sweep's panel gather
  cudaStream_t stream2 = nullptr;
  cudaEvent_t ev_pack = nullptr, ev_cold = nullptr;
  bool cold_pending = false;                 // ev_cold has been recorded and not yet waited for by a main sweep

  void* peer_xt[2][LUXB_MAX_PARTS]{};
  bool replica_stale = false;                // natural-order replica holds only this rank's slice (gathered on demand)
  // push apps
  uint32_t* d_cur = nullptr;       // [n_part] working labels of this partition
  uint64_t* d_out_end = nullptr;   // [nv] CSR-by-source end offsets over this partition's edges
  uint32_t* d_out_dst = nullptr;   // [e_part]
  int32_t* d_out_w = nullptr;      // [e_part] weighted SSSP: the weight of each out-edge, aligned with d_out_dst
  void* d_big_list = nullptr;      // segments of hub sources' out-edge lists (push_big_kernel)
  uint32_t big_capacity = 0;
  unsigned char* d_fq_all = nullptr;  // every partition's frontier slot as exchanged
  unsigned char* d_fq_new = nullptr;  // this partition's slot under construction
  unsigned char* d_fq_tmp = nullptr;
  uint32_t* d_hdr_all = nullptr;      // [2 * P] gathered headers
  luxb::FrontierCtl* d_fctl = nullptr;  // device-side frontier finalisation flags (push.cuh)
  uint64_t* d_slot_off = nullptr;
  uint32_t* h_hdr = nullptr;          // pinned [2 * P]: type, count of the current frontier of every partition
  uint32_t* h_scratch = nullptr;      // pinned scratch (header readback)
  unsigned long long* d_counters = nullptr;  // [0] edges scanned by push kernels, [1] check mistakes
  CfState cf;
  BcState bc;
  TcState tc;
  KcoreState kc;
  TrussState tr;

  // communication
  luxb::ncclComm_t comm = nullptr;
  bool p2p_ready = false;
  void* peer_val[2][LUXB_MAX_PARTS]{};  // imported replicas of the peers (P2P exchange)
  void* peer_fq[LUXB_MAX_PARTS]{};      // imported frontier slot tables of the peers (CC / SSSP P2P push)
  uint32_t* d_sync = nullptr;
  // iteration barrier of the P2P paths without a library call: every rank owns P flag words, peers store their barrier
  // epoch into "their" word over NVLink and spin on their own (flag_barrier_kernel, build.cuh)
  uint32_t* d_flags = nullptr;
  void* peer_flags[LUXB_MAX_PARTS]{};
  uint32_t barrier_epoch = 0;
  uint32_t* h_barrier_err = nullptr;  // mapped pinned word: set when a peer did not arrive in time
  uint64_t barrier_timeout_ns = 30000000000ull;
  bool flag_barrier = true;           // LUXB_BARRIER=nccl: the 4-byte all-reduce of the communicator instead
  bool flag_barrier_all = false;      // LUXB_BARRIER=flag: also for the CC / SSSP / col_filter barriers
  bool direct_push = false;           // LUXB_PUSH=direct: owners store into EVERY rank's transfer array, no chunk pulls

  SweepSettings sweep;

  // source-blocked PageRank sweep (panel.cuh): hub destinations x hot source blocks in shared memory
  bool empties_done[2] = {false, false};  // value buffer k already holds update(identity) at the edge-less vertices
  bool seg_on = false;             // PageRank sweeps the flagged stream(s) of seg.cuh (sb_main [+ sb_panel])
  bool sb_on = false;
  PullLayout sb_main, sb_panel;
  uint32_t sb_n_hub = 0, sb_n_blocks = 0, sb_n_groups = 0, sb_bs = 0;  // groups: sb_n_blocks panel blocks, then cold segments
  uint32_t* d_hub_vtx = nullptr;
  uint32_t* d_hub_bits = nullptr;
  uint32_t* d_sb_partial = nullptr;  // [slots] raw reductions of every (group, hub) pair with edges (4-byte Acc)
  uint32_t* d_slot_bits = nullptr;   // [wbase[sb_n_groups]] which (group, hub) pairs have a slot (panel.cuh)
  uint32_t* d_slot_pre = nullptr;    // [wbase[sb_n_groups] + 1] slots before each bitmap word
  luxb::SplitGroups sb_groups{};
  uint32_t sb_super_end[luxb::kPanelMaxBlocks]{};
  // cold-hub stream (PageRank, one rank): cold source segment x hub destination, gathered through L1 from an L2-sized
  // segment of the compact cold values (panel.cuh, ColdSplit)
  bool cold_z = false;             // one rank: d_hot = Z = [hot copies | cold-active values in id order], d_hot_order covers both
  bool cs_on = false;
  PullLayout sb_cold;
  // concurrent split sweep (one rank, sb_on): the cold-hub and main kernels on stream_b beside the panel kernel on
  // `stream`; ev_fork / ev_join hand the sweep over and back
  cudaStream_t stream_b = nullptr;
  cudaEvent_t ev_fork = nullptr, ev_join = nullptr;

  // launch configuration resolved once at open time (no getenv / function-static state on the hot path)
  int pull_ctas = 3;
  bool overlap_exchange = true;  // cold half of the PageRank exchange on the second stream (LUXB_OVERLAP=0: serialised)
  bool fused_fixup = true;  // one chained-scan launch instead of the three fix-up kernels (LUXB_FUSED_FIXUP=0: three)
  int panel_reserve_sms = 12;  // SMs the panel kernel leaves to the overlapped collective on several ranks
  int l2_hints = 1;   // LUXB_L2_HINTS: per-gather L2 eviction policies in the L1 sweep (hot evict_last, cold evict_first)
  PhaseTimer pt;

  // optional per-launch timing of the dominant kernel
  bool kernel_timing = false;
  std::vector<cudaEvent_t> kt_events;  // pairs
  size_t kt_used = 0;

  std::vector<OwnedBuf> owned;  // every buffer above, in order of allocation (api.cu: gmalloc); luxb_close frees them

  // stats / trace
  luxb_stats_t stats{};
  std::vector<uint64_t> trace_active;
  std::vector<int32_t> trace_pull;
};
