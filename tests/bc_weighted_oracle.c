/*
 * bc_weighted_oracle.c — CPU oracle of weighted betweenness centrality (test infrastructure, NOT product code; the
 * product never links it).
 *
 * Restates the semantics of LUXB_BC_WEIGHTED (include/lux_b200.h) in plain C + OpenMP as Brandes' algorithm over
 * shortest-path distances.  To stay independent of the device algorithm (Jacobi label iterations, then a sort of the
 * distances), the distances come from a binary-heap Dijkstra per source.  It is pinned by independent implementations:
 * tests/test_bc_weighted_oracle.py compares it with networkx, scipy's Dijkstra, the weighted SSSP oracle, the unweighted
 * BC oracle (unit weights, bit for bit) and hand-worked graphs.  Semantics:
 *   the graph is the CSC's directed edges u -> v (one per in-edge of v) with i32 weights w, every w >= 1;
 *   D[v]     = distance from s, u32, sat_add(D[u], w) = min(D[u] + w, INF), INF = 2^32 - 1 (a sum reaching INF is
 *              unreachable);
 *   tight    : (u, v, w) with D[v] != INF and (uint64)D[u] + w == D[v];
 *   sigma[s] = 1, sigma[v] = sum of sigma[u] over the tight in-edges of v (multiplicity counts, a self-loop never
 *              matches since w >= 1);
 *   delta[v] = sigma[v] * sum of t[x] over the tight out-edges (v, x), t[x] = (1 + delta[x]) / sigma[x];
 *   unreachable vertices: sigma = delta = 0;  scores[v] += delta[v] for every source s != v, sources in list order.
 * Vertices are processed in ascending distance (one class per distinct distance, ids ascending inside it).  Every
 * vertex's sum runs over its edges in CSC order (in-edges) or CSR order (out-edges, destinations ascending), exactly as
 * in bc_oracle.c, so unit weights reproduce it bit for bit; the vertices of one class are independent, so the OpenMP
 * loops leave every result deterministic.
 */
#include <stdint.h>
#include <stdlib.h>
#include <string.h>
#ifdef _OPENMP
#include <omp.h>
#endif

typedef uint32_t V_ID;
typedef uint64_t E_ID;
#define BWO_INF 0xFFFFFFFFu

typedef struct {
  V_ID nv;
  const E_ID* row_end;  /* CSC: in-edges of v are src[row_end[v-1] .. row_end[v]) with weights w[..] */
  const V_ID* src;
  const int32_t* w;
  E_ID* out_beg;        /* CSR: out-edges of u are out_dst[out_beg[u] .. out_beg[u+1]), weights out_w */
  V_ID* out_dst;
  int32_t* out_w;
  V_ID* order;          /* reached vertices by (D, id); class k is order[cls[k] .. cls[k+1]) */
  V_ID* cls;
  V_ID* heap;           /* Dijkstra: binary min-heap of vertices keyed by (D, id), pos[v] = index or -1 */
  int64_t* pos;
} bwo_graph;

static E_ID in_beg(const bwo_graph* g, V_ID v) { return v ? g->row_end[v - 1] : 0; }

static inline V_ID sat_add(V_ID d, int32_t w) {
  uint64_t s = (uint64_t)d + (uint32_t)w;
  return s < BWO_INF ? (V_ID)s : BWO_INF;
}

static inline int tight(V_ID from, int32_t w, V_ID to) { return to != BWO_INF && (uint64_t)from + (uint32_t)w == to; }

static int bwo_build(bwo_graph* g, V_ID nv, E_ID ne, const E_ID* row_end, const V_ID* src, const int32_t* w) {
  memset(g, 0, sizeof(*g));
  g->nv = nv;
  g->row_end = row_end;
  g->src = src;
  g->w = w;
  g->out_beg = (E_ID*)calloc((size_t)nv + 1, sizeof(E_ID));
  g->out_dst = (V_ID*)malloc((ne ? ne : 1) * sizeof(V_ID));
  g->out_w = (int32_t*)malloc((ne ? ne : 1) * sizeof(int32_t));
  g->order = (V_ID*)malloc(((size_t)nv + 1) * sizeof(V_ID));
  g->cls = (V_ID*)malloc(((size_t)nv + 2) * sizeof(V_ID));
  g->heap = (V_ID*)malloc(((size_t)nv + 1) * sizeof(V_ID));
  g->pos = (int64_t*)malloc(((size_t)nv + 1) * sizeof(int64_t));
  E_ID* cur = (E_ID*)malloc(((size_t)nv + 1) * sizeof(E_ID));
  if (!g->out_beg || !g->out_dst || !g->out_w || !g->order || !g->cls || !g->heap || !g->pos || !cur) { free(cur); return -1; }
  for (E_ID e = 0; e < ne; ++e) g->out_beg[src[e] + 1]++;
  for (V_ID u = 0; u < nv; ++u) g->out_beg[u + 1] += g->out_beg[u];
  memcpy(cur, g->out_beg, ((size_t)nv + 1) * sizeof(E_ID));
  for (V_ID v = 0; v < nv; ++v)  /* destinations visited in ascending order: each out-list is ascending */
    for (E_ID e = in_beg(g, v); e < row_end[v]; ++e) {
      E_ID k = cur[src[e]]++;
      g->out_dst[k] = v;
      g->out_w[k] = w[e];
    }
  free(cur);
  return 0;
}

static void bwo_free(bwo_graph* g) {
  free(g->out_beg);
  free(g->out_dst);
  free(g->out_w);
  free(g->order);
  free(g->cls);
  free(g->heap);
  free(g->pos);
}

/* ---- Dijkstra with an indexed binary heap ---------------------------------------------------------------------- */
static inline int before(const V_ID* D, V_ID a, V_ID b) { return D[a] < D[b] || (D[a] == D[b] && a < b); }

static void heap_up(bwo_graph* g, const V_ID* D, int64_t i) {
  V_ID v = g->heap[i];
  while (i > 0) {
    int64_t p = (i - 1) / 2;
    if (!before(D, v, g->heap[p])) break;
    g->heap[i] = g->heap[p];
    g->pos[g->heap[i]] = i;
    i = p;
  }
  g->heap[i] = v;
  g->pos[v] = i;
}

static void heap_down(bwo_graph* g, const V_ID* D, int64_t i, int64_t n) {
  V_ID v = g->heap[i];
  for (;;) {
    int64_t c = 2 * i + 1;
    if (c >= n) break;
    if (c + 1 < n && before(D, g->heap[c + 1], g->heap[c])) ++c;
    if (!before(D, g->heap[c], v)) break;
    g->heap[i] = g->heap[c];
    g->pos[g->heap[i]] = i;
    i = c;
  }
  g->heap[i] = v;
  g->pos[v] = i;
}

/* D of every vertex; order[] = the reached vertices in pop order, which is (D, id) ascending; returns their number */
static V_ID dijkstra(bwo_graph* g, V_ID s, V_ID* D) {
  const V_ID nv = g->nv;
  for (V_ID v = 0; v < nv; ++v) { D[v] = BWO_INF; g->pos[v] = -1; }
  D[s] = 0;
  int64_t n = 0;
  g->heap[n++] = s;
  g->pos[s] = 0;
  V_ID reached = 0;
  while (n > 0) {
    V_ID u = g->heap[0];
    g->pos[u] = -2;  /* settled */
    g->order[reached++] = u;
    if (--n > 0) { g->heap[0] = g->heap[n]; g->pos[g->heap[0]] = 0; heap_down(g, D, 0, n); }
    for (E_ID e = g->out_beg[u]; e < g->out_beg[u + 1]; ++e) {
      V_ID x = g->out_dst[e];
      V_ID c = sat_add(D[u], g->out_w[e]);
      if (c < D[x]) {  /* INF never improves: a saturated sum leaves x unreached */
        D[x] = c;
        if (g->pos[x] == -1) { g->heap[n] = x; g->pos[x] = n; ++n; }
        heap_up(g, D, g->pos[x]);
      }
    }
  }
  return reached;
}

/* one source; returns the number of distance classes */
static V_ID bwo_source(bwo_graph* g, V_ID s, V_ID* D, double* sigma, double* delta) {
  const V_ID nv = g->nv;
  for (V_ID v = 0; v < nv; ++v) { sigma[v] = 0.0; delta[v] = 0.0; }
  const V_ID reached = dijkstra(g, s, D);
  V_ID C = 0;
  for (V_ID i = 0; i < reached; ++i)
    if (i == 0 || D[g->order[i - 1]] != D[g->order[i]]) g->cls[C++] = i;
  g->cls[C] = reached;
  sigma[s] = 1.0;
  for (V_ID k = 1; k < C; ++k) {
    const int64_t a = g->cls[k], b = g->cls[k + 1];
#pragma omp parallel for schedule(dynamic, 64) if (b - a > 256)
    for (int64_t i = a; i < b; ++i) {
      V_ID v = g->order[i];
      double sum = 0.0;
      for (E_ID e = in_beg(g, v); e < g->row_end[v]; ++e)
        if (tight(D[g->src[e]], g->w[e], D[v])) sum += sigma[g->src[e]];
      sigma[v] = sum;
    }
  }
  for (V_ID k = C - 1; k >= 1; --k) {  /* delta of class k - 1 from the larger classes */
    const int64_t a = g->cls[k - 1], b = g->cls[k];
#pragma omp parallel for schedule(dynamic, 64) if (b - a > 256)
    for (int64_t i = a; i < b; ++i) {
      V_ID v = g->order[i];
      double sum = 0.0;
      for (E_ID e = g->out_beg[v]; e < g->out_beg[v + 1]; ++e) {
        V_ID x = g->out_dst[e];
        if (tight(D[v], g->out_w[e], D[x])) sum += (1.0 + delta[x]) / sigma[x];
      }
      delta[v] = sigma[v] * sum;
    }
  }
  return C;
}

/* Process the sources in order: scores (if not NULL, [nv], not cleared) += delta_s at every v != s; dist / sigma / delta
 * ([nv] each, caller-owned) end as the last source's state, classes_out[i] = distance classes of source i.  Returns 0,
 * -1 when out of memory or a source >= nv, -2 when a weight is < 1 (nothing is computed). */
int bwo_run(V_ID nv, E_ID ne, const E_ID* row_end, const V_ID* src, const int32_t* w, const V_ID* sources, int n_sources,
            double* scores, V_ID* dist, double* sigma, double* delta, V_ID* classes_out) {
  for (E_ID e = 0; e < ne; ++e)
    if (w[e] < 1) return -2;
  for (int i = 0; i < n_sources; ++i)
    if (sources[i] >= nv) return -1;
  bwo_graph g;
  if (bwo_build(&g, nv, ne, row_end, src, w)) { bwo_free(&g); return -1; }
  for (int i = 0; i < n_sources; ++i) {
    V_ID s = sources[i];
    V_ID C = bwo_source(&g, s, dist, sigma, delta);
    if (classes_out) classes_out[i] = C;
    if (scores) {
#pragma omp parallel for schedule(static)
      for (int64_t v = 0; v < (int64_t)nv; ++v)
        if ((V_ID)v != s) scores[v] += delta[v];
    }
  }
  bwo_free(&g);
  return 0;
}
