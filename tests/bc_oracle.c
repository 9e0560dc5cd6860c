/*
 * bc_oracle.c — CPU oracle of betweenness centrality (test infrastructure, NOT product code; the product never links it).
 *
 * The reference has no betweenness centrality, so nothing can be replayed: this restates the semantics of LUXB_BC
 * (include/lux_b200.h) in plain C + OpenMP as Brandes' algorithm.  It is pinned by independent implementations:
 * tests/test_bc_oracle.py compares it with networkx and with hand-worked graphs.  Semantics:
 *   the graph is the CSC's directed edges u -> v (one per in-edge of v), unweighted;
 *   lev[v]   = hop distance from s (INF = nv), found by a level-synchronous BFS over the out-edges;
 *   sigma[s] = 1, sigma[v] = sum of sigma[u] over in-edges (u, v) with lev[u] = lev[v] - 1 (multiplicity counts, a
 *              self-loop never matches);
 *   delta[v] = sigma[v] * sum of t[w] over out-edges (v, w) with lev[w] = lev[v] + 1, t[w] = (1 + delta[w]) / sigma[w];
 *   unreachable vertices: sigma = delta = 0;  scores[v] += delta[v] for every source s != v, sources in list order.
 * Every vertex's sum runs over its edges in CSC order (in-edges) or CSR order (out-edges, destinations ascending);
 * the vertices of one level are independent, so the OpenMP loops leave every result deterministic.
 */
#include <stdint.h>
#include <stdlib.h>
#include <string.h>
#ifdef _OPENMP
#include <omp.h>
#endif

typedef uint32_t V_ID;
typedef uint64_t E_ID;

typedef struct {
  V_ID nv;
  const E_ID* row_end;  /* CSC: in-edges of v are src[row_end[v-1] .. row_end[v]) */
  const V_ID* src;
  E_ID* out_beg;        /* CSR: out-edges of u are out_dst[out_beg[u] .. out_beg[u+1]) */
  V_ID* out_dst;
  V_ID* queue;          /* BFS order: the vertices of level d are queue[lev_off[d] .. lev_off[d+1]) */
  V_ID* lev_off;
} bco_graph;

static E_ID in_beg(const bco_graph* g, V_ID v) { return v ? g->row_end[v - 1] : 0; }

static int bco_build(bco_graph* g, V_ID nv, E_ID ne, const E_ID* row_end, const V_ID* src) {
  memset(g, 0, sizeof(*g));
  g->nv = nv;
  g->row_end = row_end;
  g->src = src;
  g->out_beg = (E_ID*)calloc((size_t)nv + 1, sizeof(E_ID));
  g->out_dst = (V_ID*)malloc((ne ? ne : 1) * sizeof(V_ID));
  g->queue = (V_ID*)malloc(((size_t)nv + 1) * sizeof(V_ID));
  g->lev_off = (V_ID*)malloc(((size_t)nv + 2) * sizeof(V_ID));
  E_ID* cur = (E_ID*)malloc(((size_t)nv + 1) * sizeof(E_ID));
  if (!g->out_beg || !g->out_dst || !g->queue || !g->lev_off || !cur) { free(cur); return -1; }
  for (E_ID e = 0; e < ne; ++e) g->out_beg[src[e] + 1]++;
  for (V_ID u = 0; u < nv; ++u) g->out_beg[u + 1] += g->out_beg[u];
  memcpy(cur, g->out_beg, ((size_t)nv + 1) * sizeof(E_ID));
  for (V_ID v = 0; v < nv; ++v)  /* destinations visited in ascending order: each out-list is ascending */
    for (E_ID e = in_beg(g, v); e < row_end[v]; ++e) g->out_dst[cur[src[e]]++] = v;
  free(cur);
  return 0;
}

static void bco_free(bco_graph* g) {
  free(g->out_beg);
  free(g->out_dst);
  free(g->queue);
  free(g->lev_off);
}

/* one source; returns the number of levels L */
static V_ID bco_source(bco_graph* g, V_ID s, V_ID* lev, double* sigma, double* delta) {
  const V_ID nv = g->nv;
  for (V_ID v = 0; v < nv; ++v) { lev[v] = nv; sigma[v] = 0.0; delta[v] = 0.0; }
  lev[s] = 0;
  g->queue[0] = s;
  g->lev_off[0] = 0;
  V_ID L = 0, head = 0, tail = 1;
  while (head < tail) {  /* level L is queue[head .. tail) */
    g->lev_off[L] = head;
    V_ID end = tail;
    for (V_ID i = head; i < end; ++i) {
      V_ID u = g->queue[i];
      for (E_ID e = g->out_beg[u]; e < g->out_beg[u + 1]; ++e) {
        V_ID w = g->out_dst[e];
        if (lev[w] == nv) { lev[w] = L + 1; g->queue[tail++] = w; }
      }
    }
    head = end;
    ++L;
  }
  g->lev_off[L] = tail;
  sigma[s] = 1.0;
  for (V_ID d = 1; d < L; ++d) {
    const int64_t a = g->lev_off[d], b = g->lev_off[d + 1];
#pragma omp parallel for schedule(dynamic, 64)
    for (int64_t i = a; i < b; ++i) {
      V_ID v = g->queue[i];
      double sum = 0.0;
      for (E_ID e = in_beg(g, v); e < g->row_end[v]; ++e)
        if (lev[g->src[e]] == d - 1) sum += sigma[g->src[e]];
      sigma[v] = sum;
    }
  }
  for (V_ID d = L - 1; d >= 1; --d) {  /* delta of level d - 1 from level d */
    const int64_t a = g->lev_off[d - 1], b = g->lev_off[d];
#pragma omp parallel for schedule(dynamic, 64)
    for (int64_t i = a; i < b; ++i) {
      V_ID v = g->queue[i];
      double sum = 0.0;
      for (E_ID e = g->out_beg[v]; e < g->out_beg[v + 1]; ++e) {
        V_ID w = g->out_dst[e];
        if (lev[w] == d) sum += (1.0 + delta[w]) / sigma[w];
      }
      delta[v] = sigma[v] * sum;
    }
  }
  return L;
}

/* Process the sources in order: scores (if not NULL, [nv], not cleared) += delta_s at every v != s; lev / sigma / delta
 * ([nv] each, caller-owned) end as the last source's state.  Returns 0, or -1 when out of memory or a source >= nv. */
int bco_run(V_ID nv, E_ID ne, const E_ID* row_end, const V_ID* src, const V_ID* sources, int n_sources, double* scores,
            V_ID* lev, double* sigma, double* delta, V_ID* levels_out) {
  for (int i = 0; i < n_sources; ++i)
    if (sources[i] >= nv) return -1;
  bco_graph g;
  if (bco_build(&g, nv, ne, row_end, src)) { bco_free(&g); return -1; }
  for (int i = 0; i < n_sources; ++i) {
    V_ID s = sources[i];
    V_ID L = bco_source(&g, s, lev, sigma, delta);
    if (levels_out) levels_out[i] = L;
    if (scores) {
#pragma omp parallel for schedule(static)
      for (int64_t v = 0; v < (int64_t)nv; ++v)
        if ((V_ID)v != s) scores[v] += delta[v];
    }
  }
  bco_free(&g);
  return 0;
}
