/*
 * lux_b200.h — C ABI of the H100-native Lux hot path (libluxb.so).
 *
 * The reference (LuxGraph/Lux) has no C ABI: its plugin boundary is the list of Legion task bodies that
 * core/graph.h declares and each <app>_gpu.cu defines.  Every entry point below replaces one of those task
 * bodies (or one phase of an app's top_level_task) with a Legion-free call taking plain pointers and sizes.
 * Reference citations are file:line inside /root/reference.
 *
 * Model: ONE PROCESS PER GPU.  A handle (luxb_graph) is one rank's view: the global partition table plus the
 * rank's own destination-vertex range [row_left, row_right], its CSC slice in HBM (and, for push apps, the
 * CSR-by-source index of the same edges), a full replica of the vertex-value array, and the exchange machinery
 * (NCCL all-gather or direct peer-HBM stores).  With nranks == 1 no communication library is touched.
 *
 * Conventions: every function returns 0 on success and a negative luxb_status on failure; luxb_last_error()
 * returns a thread-local message.  Nothing calls exit()/assert() on bad input (the reference does:
 * core/cuda_helper.h:6-20).  A handle may be used by one host thread at a time.
 */
#ifndef LUX_B200_H_
#define LUX_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef uint32_t luxb_vid; /* V_ID  — pagerank/app.h:21 */
typedef uint64_t luxb_eid; /* E_ID  — pagerank/app.h:22 */

#define LUXB_MAX_PARTS 64          /* MAX_NUM_PARTS — core/graph.h:31 */
#define LUXB_CF_K 20               /* K — col_filter/app.h:28 */
#define LUXB_DENSE_BITMAP 0x1234567u /* FrontierHeader::DENSE_BITMAP — core/graph.h:102 */
#define LUXB_SPARSE_QUEUE 0x7654321u /* FrontierHeader::SPARSE_QUEUE — core/graph.h:103 */
#define LUXB_UNIQUE_ID_BYTES 128   /* sizeof(ncclUniqueId) */

typedef enum {
  LUXB_OK = 0,
  LUXB_ERR_ARG = -1,      /* bad argument / malformed graph */
  LUXB_ERR_CUDA = -2,     /* CUDA runtime error (message has the CUDA string) */
  LUXB_ERR_IO = -3,       /* file could not be read */
  LUXB_ERR_COMM = -4,     /* NCCL / peer-memory error */
  LUXB_ERR_STATE = -5,    /* call out of order (e.g. iterate before init) */
  LUXB_ERR_NOMEM = -6
} luxb_status;

typedef enum {
  LUXB_PAGERANK = 0, /* pagerank/   — pull model, f32 vertex value (rank / out-degree) */
  LUXB_CC = 1,       /* components/ — push/pull hybrid, u32 label, max */
  LUXB_SSSP = 2,     /* sssp/       — push/pull hybrid, u32 hop distance, min(+1), INF = nv */
  LUXB_COLFILTER = 3, /* col_filter/ — pull model, float[20] vertex value */
  LUXB_SSSP_WEIGHTED = 4, /* weighted SSSP (no reference counterpart) — push/pull hybrid, u32 distance, INF = LUXB_DIST_INF */
  LUXB_BC = 5,           /* betweenness centrality (no reference counterpart) — Brandes over the SSSP engine's hop levels,
                            f64 score per vertex; runs through luxb_bc_run */
  LUXB_BC_WEIGHTED = 6,  /* weighted betweenness centrality (no reference counterpart) — Brandes over the weighted SSSP
                            distances (weights >= 1), f64 score per vertex; runs through luxb_bc_run */
  LUXB_TC = 7            /* triangle counting (no reference counterpart) — exact u64 count of the triangles at every
                            vertex of the undirected simple graph; runs through luxb_tc_run */
} luxb_app;

/* Weighted SSSP (LUXB_SSSP_WEIGHTED):
 *  - weights are the CSC's i32 per-edge weights, in CSC edge order; they must be >= 0 (zero is allowed): a negative
 *    weight fails the open with LUXB_ERR_ARG.  The graph must carry weights (csc->weight, or the .lux i32 trailer);
 *    luxb_open_rmat generates them (see there), luxb_open_bipartite uses its ratings 1..5;
 *  - distances are u32; INF = LUXB_DIST_INF (not nv: real distances can exceed nv).  D[start] = 0, every other INF;
 *  - relaxation cand = sat_add(D[u], w) = min(D[u] + w, INF), computed without wrap-around: INF + w = INF, and a
 *    distance that would reach 2^32 - 1 reads as unreachable;
 *  - otherwise SSSP's structure: Jacobi iterations, pull when the global active count > nv/16 (the merge-path sweep),
 *    push otherwise, the same frontier representation rules, halt on zero active.  Labels after every iteration do not
 *    depend on the direction taken, so labels, per-iteration active counts and pull flags are deterministic;
 *  - luxb_check counts the in-edges with D[u] != INF && D[v] > sat_add(D[u], w).
 * LUXB_SSSP keeps its hop-count semantics even when the CSC passed to it carries weights. */
#define LUXB_DIST_INF 0xFFFFFFFFu

/* Betweenness centrality (LUXB_BC).  The graph is the CSC's directed edges u -> v, one per in-edge of v; paths are
 * unweighted (weights are ignored).  For a source s:
 *  - lev[v] is the hop distance exactly as LUXB_SSSP computes it; INF = nv for unreachable vertices;
 *  - sigma[s] = 1; every other sigma[v] = sum of sigma[u] over the in-edges (u, v) with lev[u] = lev[v] - 1 (fp64).
 *    Parallel edges count with their multiplicity; a self-loop never matches;
 *  - delta[v] = sigma[v] * sum of t[w] over the out-edges (v, w) with lev[w] = lev[v] + 1, t[w] = (1 + delta[w]) / sigma[w];
 *  - unreachable vertices have sigma = delta = 0.
 * For a list of sources S: BC[v] = sum over s in S, s != v, of delta_s(v), in fp64, not normalised; a source listed twice
 * counts twice.  S = all vertices gives exact directed BC, a sample the usual estimate; on a graph stored with both
 * directions of every edge the scores are twice the undirected BC.
 * A BC handle's values (luxb_get_values / luxb_set_values and the _local_ variants) are the scores, 8 bytes per vertex.
 * luxb_iterate, luxb_run_to_convergence and luxb_check return LUXB_ERR_ARG on it.  luxb_stats: iterations /
 * pull_iterations = BFS iterations summed over sources, edges_processed = BFS scans + sigma edges + delta edges,
 * loop_seconds = device time of the luxb_bc_run calls.  luxb_trace holds the BFS trace of the last source only. */

/* Weighted betweenness centrality (LUXB_BC_WEIGHTED).  The graph is the CSC's directed edges u -> v with their i32
 * weights w, and every weight must be >= 1: a smaller one fails the open with LUXB_ERR_ARG (checked on the device).  With
 * w >= 1 every shortest-path edge goes to a strictly larger distance, so ascending distances order the shortest-path DAG;
 * a zero weight would put DAG edges inside one distance and a zero-weight cycle would make sigma unbounded.  The graph
 * must carry weights (csc->weight, or the .lux i32 trailer); luxb_open_rmat generates the [1, 255] weights of weighted
 * SSSP.  For a source s:
 *  - D[v] is the distance exactly as LUXB_SSSP_WEIGHTED computes it (u32, sat_add, INF = LUXB_DIST_INF: a path whose
 *    sum would reach 2^32 - 1 counts as unreachable);
 *  - an edge (u, v, w) is tight iff D[v] != INF and (uint64)D[u] + w == D[v], in 64 bits: an unreached u never matches,
 *    and neither does an edge whose sum saturates to INF;
 *  - sigma[s] = 1; every other sigma[v] = sum of sigma[u] over the tight in-edges of v (fp64).  Parallel edges count
 *    with their multiplicity, but only those at the minimal weight are tight; a self-loop is never tight;
 *  - delta[v] = sigma[v] * sum of t[x] over the tight out-edges (v, x), t[x] = (1 + delta[x]) / sigma[x];
 *  - unreachable vertices have sigma = delta = 0.
 * Scores accumulate as for LUXB_BC (sum over s in S, s != v, fp64, not normalised, repeats count).  Unit weights give
 * LUXB_BC exactly: D = lev, and sigma, delta and the scores are bit for bit equal.  luxb_bc_source_state returns D as
 * `lev`.  Values, luxb_iterate / luxb_run_to_convergence / luxb_check, luxb_stats and the phase timing behave as for
 * LUXB_BC; luxb_trace holds the weighted SSSP trace of the last source. */

/* Triangle counting (LUXB_TC).  The CSC's directed edges are read as an undirected simple graph: {u, v} is an edge iff
 * u != v and at least one of u -> v or v -> u is stored.  Parallel edges, both directions and self-loops collapse to that
 * one edge; weights are ignored (a weighted CSC is accepted).  A triangle is a set of three distinct, pairwise adjacent
 * vertices.
 *  - t[v] is the number of triangles that contain v, u64 (networkx's triangles() on the simple graph);
 *  - the total T = sum of t / 3, u64;
 *  - integers only: the results depend neither on the schedule nor on the number of ranks or the split.
 * luxb_init builds the oriented adjacency once (every rank holds the whole graph: its slice's edges are exchanged at
 * luxb_init); luxb_open_* read the input edges once, as for every app.  The handle's values (luxb_get_values /
 * luxb_get_local_values) are t, 8 bytes per vertex: zeros before the first luxb_tc_run, complete on every rank after one
 * (the get calls are not collective).  luxb_set_values / luxb_set_local_values, luxb_iterate, luxb_run_to_convergence and
 * luxb_check return LUXB_ERR_ARG.  luxb_stats: iterations = luxb_tc_run calls, edges_processed += m (undirected simple
 * edges) per call, loop_seconds = device time of the luxb_tc_run calls.  luxb_get_local_csc / luxb_device_view keep
 * returning this rank's CSC slice.  cfg.start_vtx, cfg.exchange and cfg.verbose have no effect. */

typedef enum {
  LUXB_EXCHANGE_NCCL = 0, /* library collectives only: PageRank packs its share and broadcasts the two ranges of every
                             owner (grouped ncclBroadcast); CC / SSSP broadcast frontier slots and label slices;
                             col_filter all-gathers the vector slices.  Needs no peer mappings */
  LUXB_EXCHANGE_P2P = 1,  /* peer memory over NVLink (luxb_p2p_export / import): PageRank = pack+push to the equal-chunk
                             holders, flag barrier kernel (system-scope release / acquire on peer flag words),
                             chunk pull — a balanced all-gather without a library call, cold half overlapped on a
                             second stream; CC / SSSP = frontier P2P push into the peers' slot tables
                             and label replicas; col_filter = peer stores of the new vectors */
  LUXB_EXCHANGE_P2P_FUSED = 2 /* kept for source compatibility: same as LUXB_EXCHANGE_P2P (round 1's fused stores from the
                             gather kernel lost at 8 GPUs and are gone) */
} luxb_exchange;

/* Whole-graph CSC in caller-owned host memory — the arrays of a .lux file (tools/converter.cc:98-124):
 * row_end[v] = END offset of v's in-edge block (row_end[nv-1] == ne, non-decreasing: pull_model.inl:99-102),
 * src[e] = source vertex of in-edge e, weight[e] optional (EDGE_WEIGHT apps, pull_model.inl:309-317). */
typedef struct {
  luxb_vid nv;
  luxb_eid ne;
  const luxb_eid* row_end;
  const luxb_vid* src;
  const int32_t* weight; /* needed by LUXB_COLFILTER, LUXB_SSSP_WEIGHTED and LUXB_BC_WEIGHTED; ignored by the others */
} luxb_csc;

typedef struct {
  luxb_app app;
  int rank;            /* this process's partition index, 0..nranks-1 (Legion point of the index launch) */
  int nranks;          /* number of partitions == number of GPUs (-ng / -ll:gpu, pagerank.cc:121-148) */
  int device;          /* CUDA device ordinal for this rank (LuxMapper::slice_task, lux_mapper.cc:97-144) */
  luxb_vid start_vtx;  /* SSSP -start (sssp.cc) */
  luxb_exchange exchange;
  int verbose;         /* -verbose: per-iteration line like components_gpu.cu:516-518 */
  int balanced_split;  /* pull apps on several ranks: 1 = split the destination range by estimated sweep cost instead of
                          by edge count (contiguous ranges, only the cut points move; results depend on the split only
                          through float summation order).  luxb_partition_bounds keeps reporting the reference's split,
                          luxb_work_bounds the one in use.  0 = the reference's split is the work split. */
  int zero_copy_edges; /* 1: keep the edge arrays (source ids, weights) in mapped pinned HOST memory and stream them
                          over PCIe every iteration — the analogue of Legion's -ll:zsize zero-copy memory for
                          graphs larger than HBM (lux_mapper.cc:146-165); vertex arrays stay in HBM */
} luxb_config;

typedef struct luxb_graph luxb_graph; /* opaque; owns all device memory (Graph + GraphPiece, core/graph.h:54-98) */

/* ---- Graph::Graph + *LoadTask: build the partition table and put this rank's slice into HBM ------------- */
/* = Graph::Graph (pull_model.inl:29-191 / push_model.inl:301-509) + pull/push_load_task_impl
 *   (pull_model.inl:253-320 / push_model.inl:78-121) reading from memory instead of a file. */
int luxb_open_csc(const luxb_csc* csc, const luxb_config* cfg, luxb_graph** out);
/* Same from a .lux file; reads header + row_end, partitions, then fseeks to this rank's slice exactly like
 * pull_load_task_impl (pull_model.inl:294-318). */
int luxb_open_file(const char* lux_path, const luxb_config* cfg, luxb_graph** out);
/* Synthetic inputs generated ON THE DEVICE (no reference counterpart; SURVEY §8d): deterministic counter-based
 * RMAT (a,b,c,d = .57,.19,.19,.05), endpoints >= nv rejected, canonical (dst,src)-sorted CSC.  Bit-identical to
 * oracle lo_gen_rmat_csc.  Every rank generates the edge stream and keeps only its own partition.
 * app == LUXB_SSSP_WEIGHTED or LUXB_BC_WEIGHTED: every edge also gets a directed weight in [1, 255] that depends only on
 * (seed, src, dst):
 *   w = 1 + (splitmix64(splitmix64(seed ^ 0x9E3779B97F4A7C15) ^ (dst << 32 | src)) >> 32) % 255
 * (bit-identical to the weighted-SSSP test oracle, tests/weighted_oracle.c wo_rmat_weight). */
int luxb_open_rmat(int scale, luxb_vid nv, luxb_eid ne, uint64_t seed, const luxb_config* cfg, luxb_graph** out);
/* NetFlix-like bipartite ratings graph, every rating stored in both directions (ne = 2*ratings), int weights 1..5. */
int luxb_open_bipartite(luxb_vid users, luxb_vid items, luxb_eid ratings, uint64_t seed, const luxb_config* cfg,
                        luxb_graph** out);

/* ---- .lux files (tools/converter.cc; format README.md:75, graph.h:32) — host only ---------------------------------- */
/* Write a CSC as a .lux file: u32 nv, u64 ne, u64 row_end[nv], u32 src[ne], then i32 weight[ne] when csc->weight is set
 * (what EDGE_WEIGHT apps read, pull_model.inl:309-317) or else u32 out_degree[nv] (what converter.cc:124 appends). */
int luxb_write_lux(const char* lux_path, const luxb_csc* csc);
/* = tools/converter.cc main (-nv -ne -input -output): text edge list "src dst" per edge -> .lux.  Edges are put in
 * canonical (dst, src) order (the reference's std::sort by dst leaves the order inside a destination unspecified);
 * malformed input is an error code, not an assert. */
int luxb_convert_edgelist(const char* edge_list_path, const char* lux_path, luxb_vid nv, luxb_eid ne);

/* ---- partition table (Graph::rowLeft/rowRight/fqLeft/fqRight, core/graph.h:62-63) ------------------------ */
int luxb_graph_info(const luxb_graph* g, luxb_vid* nv, luxb_eid* ne, int* nranks);
/* nranks entries each; fq_* are the frontier-slot byte ranges of push_model.inl:393-397 (NULL to skip). */
int luxb_partition_bounds(const luxb_graph* g, luxb_vid* row_left, luxb_vid* row_right, luxb_eid* col_left,
                          uint64_t* fq_left, uint64_t* fq_right);
/* The split of the destination range the ranks actually work on (== the reference's unless cfg.balanced_split);
 * returns 1 when it is the cost-balanced one. */
int luxb_work_bounds(const luxb_graph* g, luxb_vid* row_left, luxb_vid* row_right, luxb_eid* col_left);
/* The reference partitioner on host arrays, without a handle (pull_model.inl:108-131).  Returns the number of
 * partitions the greedy scan produces (may differ from P; the reference asserts equality). */
int luxb_partition_csc(luxb_vid nv, luxb_eid ne, const luxb_eid* row_end, int P, luxb_vid* row_left,
                       luxb_vid* row_right, luxb_eid* col_left);

/* ---- communicator (replaces Legion's implicit zero-copy exchange, SURVEY §2.1) --------------------------- */
int luxb_comm_unique_id(char id[LUXB_UNIQUE_ID_BYTES]);       /* rank 0; ship to the others out of band */
int luxb_comm_init(luxb_graph* g, const char id[LUXB_UNIQUE_ID_BYTES]); /* collective; no-op when nranks == 1 */
/* NCCL is bound at run time on the first of these two calls: the library named by the environment variable
 * LUXB_NCCL_LIBRARY when it is set and loads, else libnccl.so.2, else libnccl.so.  It must export ncclGetUniqueId,
 * ncclCommInitRank, ncclCommDestroy, ncclAllReduce, ncclBroadcast, ncclAllGather, ncclGroupStart, ncclGroupEnd and
 * ncclGetErrorString; one binding serves the whole process. */
/* P2P exchange: every rank exports its replica/frontier buffers (cudaIpcMemHandle), the caller all-gathers the
 * blobs (any transport) and hands the full table back. */
int luxb_p2p_export(luxb_graph* g, void* blob, size_t* blob_bytes);
int luxb_p2p_import(luxb_graph* g, const void* all_blobs, size_t blob_bytes_each);
/* Forget imported peer mappings: the P2P exchanges silently degrade to the NCCL exchange.  Call on EVERY rank when the
 * import failed on any of them (all ranks must use the same exchange). */
int luxb_p2p_disable(luxb_graph* g);
/* Unmap the peers' buffers from this process (the exchanges fall back to NCCL).  Teardown order on several ranks: every
 * rank calls luxb_p2p_disconnect, the ranks synchronise (any barrier), then each calls luxb_close — CUDA forbids freeing
 * an exported buffer while an importer still has it mapped. */
int luxb_p2p_disconnect(luxb_graph* g);

/* ---- Pull/PushInitTask (+PullScanTask): app state ------------------------------------------------------- */
/* = pull_scan_task_impl (pull_model.inl:322-345) + pull_init_task_impl (pagerank_gpu.cu:182-281,
 *   colfilter_gpu.cu:184-286) or push_init_task_impl (components_gpu.cu:614-766, sssp_gpu.cu:614-771). */
int luxb_init(luxb_graph* g);

/* ---- the hot loop ------------------------------------------------------------------------------------------ */
/* `iters` x Pull/PushAppTask incl. the exchange (pagerank.cc:109-113; pull_app_task_impl pagerank_gpu.cu:105-151,
 * colfilter_gpu.cu:106-154; push_app_task_impl components_gpu.cu:335-522).  For push apps *active_out receives
 * the global number of active vertices after the last iteration (Σ of the V_ID each partition returns). */
int luxb_iterate(luxb_graph* g, int iters, uint64_t* active_out);
/* components.cc:113-127 / sssp.cc without the sliding-window waste: iterate until an iteration reports zero
 * active vertices on every partition.  max_iters <= 0 means unbounded. */
int luxb_run_to_convergence(luxb_graph* g, int max_iters, int* iters_out);

/* ---- results / check / stats -------------------------------------------------------------------------------- */
/* Full vertex-value array (what the reference holds in dist_lr[iter%2]): nv * {4 | 4 | 80 | 8 (BC scores, TC counts)} bytes.  PageRank on
 * nranks > 1 exchanges only the values that are ever gathered each iteration and completes the full array on demand:
 * there the call is collective (every rank calls it at the same point). */
int luxb_get_values(luxb_graph* g, void* host_out, size_t bytes);
/* Overwrite the vertex values (H2D), e.g. to restart from a checkpoint; push apps: all vertices become active. */
int luxb_set_values(luxb_graph* g, const void* host_in, size_t bytes);
/* The same for THIS RANK'S partition only: (row_right - row_left + 1) values in local order — what a per-GPU task of
 * the reference touches (its own region, e.g. pull_init_task_impl writes new_pr[rowLeft..rowRight], pagerank_gpu.cu:
 * 255-259).  set: H2D of the slice, then the ranks exchange on the device exactly as after an iteration; get: D2H of the
 * slice.  nranks host buffers together move nv values over PCIe instead of nranks * nv.  Collective on nranks > 1. */
int luxb_set_local_values(luxb_graph* g, const void* host_in, size_t bytes);
int luxb_get_local_values(luxb_graph* g, void* host_out, size_t bytes);
/* CheckTask / check_kernel invariants (components_gpu.cu:768-837, sssp_gpu.cu:773-843): number of violating
 * edges over this rank's partition; PageRank / col_filter have no check in the reference -> LUXB_ERR_ARG.
 * LUXB_SSSP_WEIGHTED: in-edges with D[u] != LUXB_DIST_INF && D[v] > sat_add(D[u], w). */
int luxb_check(luxb_graph* g, uint64_t* mistakes_out);

typedef struct {
  double loop_seconds;       /* device time of iterate calls so far (the reference's ELAPSED TIME region) */
  uint64_t iterations;       /* iterations executed */
  uint64_t edges_processed;  /* PR/CF: local edges x iterations; push apps: edges actually scanned */
  uint64_t pull_iterations;  /* push apps: iterations that took the pull direction (components_gpu.cu:414) */
  uint64_t kernel_launches;  /* our kernels launched by iterate calls */
  uint64_t last_active;      /* global active count after the last iteration */
  uint32_t last_frontier_type; /* this rank's frontier representation after the last iteration */
  double dominant_kernel_seconds;   /* with kernel timing on: device time inside the gather kernel(s) only */
  uint64_t dominant_kernel_launches;
  uint64_t panel_edges;      /* PageRank: local edges swept by the source-blocked (shared-memory) kernel; 0 = plain sweep */
  uint32_t panel_hubs;       /*   hub destinations of this partition */
  uint32_t panel_blocks;     /*   hot source blocks */
  uint64_t cold_hub_edges;   /* PageRank, one rank: local (cold source -> hub) edges swept by segment of the cold values */
  uint32_t cold_hub_segments; /*   cold source segments (0 = no cold-hub stream) */
  uint32_t tier_blocks;      /* PageRank: hot source blocks after the first panel_blocks, each over a prefix of the hubs */
  uint64_t tier_slots;       /*   their (block, hub) slots */
  uint64_t tier_edges;       /*   their edges */
} luxb_stats_t;
int luxb_stats(const luxb_graph* g, luxb_stats_t* out);
/* Per-iteration trace of push apps (global active count, direction) for parity tests; returns #entries copied. */
int luxb_trace(const luxb_graph* g, uint64_t* active, int32_t* pull, int max_entries);

/* Bracket every launch of the dominant (edge gather) kernel with CUDA events on the launching stream so that the
 * bench can report its average duration for the roofline (stats.dominant_kernel_*).  Off by default. */
int luxb_enable_kernel_timing(luxb_graph* g, int on);
/* PageRank: the global out-degree array computed by the scan phase (pull_scan_task_impl, pull_model.inl:322-345). */
int luxb_get_out_degree(luxb_graph* g, luxb_vid* host_out, size_t bytes);

/* Dev tooling: time a bare gather sweep (no reduction) over this partition's source ids, natural (packed = 0) or
 * hot-packed (packed = 1) layout — the memory-system ceiling the pull kernel is compared against. */
int luxb_debug_gather_ms(luxb_graph* g, int packed, float* ms_out);

/* Raw device pointers for tooling (bench roofline timing, interop); not needed by normal callers. */
typedef struct {
  void* values;          /* replica of the current vertex values, nv entries */
  const luxb_eid* row_end; /* this rank's offsets, relative to col_left */
  const luxb_vid* src;
  void* stream;          /* cudaStream_t the hot loop runs on */
  luxb_vid row_left, row_right;
  luxb_eid local_edges;
} luxb_device_view;
int luxb_device_view_get(luxb_graph* g, luxb_device_view* out);

/* Copy this rank's CSC slice back to host (tests: generator parity).  Arrays sized from luxb_device_view. */
int luxb_get_local_csc(luxb_graph* g, luxb_eid* row_end_abs, luxb_vid* src, int32_t* weight);

/* ---- betweenness centrality (LUXB_BC and LUXB_BC_WEIGHTED handles) ------------------------------------------------ */
/* Process the sources in order and add each source's delta into the handle's scores.  Collective on nranks > 1: every rank
 * passes the same list.  Every source is validated before any work starts: a source >= nv returns LUXB_ERR_ARG and leaves
 * the scores unchanged.  n_sources == 0 is a no-op.  LUXB_ERR_STATE before luxb_init, LUXB_ERR_ARG on another app. */
int luxb_bc_run(luxb_graph* g, const luxb_vid* sources, int n_sources);
/* The full lev / sigma / delta arrays (nv_count == nv entries each) of the last source processed (LUXB_BC_WEIGHTED: lev
 * is the u32 distance D); a NULL pointer skips that array.  Every rank holds them complete: not collective.  LUXB_ERR_STATE before the first source. */
int luxb_bc_source_state(luxb_graph* g, uint32_t* lev, double* sigma, double* delta, size_t nv_count);

/* ---- triangle counting (LUXB_TC handles) --------------------------------------------------------------------------- */
/* Recount t from zero and write the total T to *total_out (may be NULL).  Every call gives the same result.  Collective on
 * nranks > 1: each rank counts the triangles found at the vertices of its own range, then t is summed over the ranks.
 * LUXB_ERR_STATE before luxb_init, LUXB_ERR_ARG on another app. */
int luxb_tc_run(luxb_graph* g, uint64_t* total_out);

void luxb_close(luxb_graph* g);
const char* luxb_last_error(void);
const char* luxb_version(void);
/* Incremented whenever the layout of a public struct changes; bindings check it before the first call. */
int luxb_abi_version(void);

#ifdef __cplusplus
}
#endif
#endif /* LUX_B200_H_ */
