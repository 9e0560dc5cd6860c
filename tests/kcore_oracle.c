// kcore_oracle.c — CPU oracle of the k-core decomposition (LUXB_KCORE), test infrastructure only.  C + OpenMP.
//
// Semantics (as in include/lux_b200.h and DESIGN §0): the CSC's directed edges are read as an undirected simple graph,
// {u, v} is an edge iff u != v and u -> v or v -> u is stored (parallel edges, both directions and self-loops collapse,
// weights are ignored).  core[v] is the largest k such that v lies in a subgraph whose every vertex has degree >= k.
//
// Two independent algorithms over the same neighbour lists (built by a counting sort over the endpoints, then sorted
// and deduplicated per vertex):
//  - Batagelj-Zaversnik bucket peeling, O(n + m): vertices kept sorted by current degree in bins; the core numbers;
//  - the level-synchronous schedule of the device, sequentially: k = 0; while a vertex is alive: k = max(k, min deg
//    over the alive vertices); repeat: F = {alive v : deg(v) <= k}, stop if F is empty, core[F] = k, remove F and lower
//    the degrees of the rest.  Its rounds, levels, per-round (|F|, k) trace, degeneracy and core numbers.
// kco_check counts the vertices that are not a fixpoint of the h-index operator (the luxb_check of LUXB_KCORE).
#include <omp.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

static int cmp_u32(const void* a, const void* b) {
  const uint32_t x = *(const uint32_t*)a, y = *(const uint32_t*)b;
  return (x > y) - (x < y);
}

typedef struct {
  uint64_t* start;  // [nv + 1] list of v at adj[start[v], start[v] + deg[v])
  uint32_t* deg;    // [nv] distinct neighbours
  uint32_t* adj;
} Graph;

static void graph_free(Graph* g) {
  free(g->start);
  free(g->deg);
  free(g->adj);
}

// 0, -1 when a source id is >= nv, -2 when out of memory
static int graph_build(uint32_t nv, const uint64_t* row_end, const uint32_t* src, Graph* g) {
  memset(g, 0, sizeof(*g));
  g->start = calloc((size_t)nv + 1, 8);
  g->deg = calloc((size_t)nv + 1, 4);
  if (!g->start || !g->deg) return -2;
  for (uint32_t v = 0; v < nv; ++v)
    for (uint64_t e = v ? row_end[v - 1] : 0; e < row_end[v]; ++e) {
      const uint32_t u = src[e];
      if (u >= nv) return -1;
      if (u == v) continue;
      g->start[u + 1]++;
      g->start[v + 1]++;
    }
  for (uint32_t v = 0; v < nv; ++v) g->start[v + 1] += g->start[v];
  g->adj = malloc((size_t)g->start[nv] * 4 + 4);
  uint64_t* fill = malloc((size_t)nv * 8 + 8);
  if (!g->adj || !fill) { free(fill); return -2; }
  memcpy(fill, g->start, (size_t)nv * 8);
  for (uint32_t v = 0; v < nv; ++v)
    for (uint64_t e = v ? row_end[v - 1] : 0; e < row_end[v]; ++e) {
      const uint32_t u = src[e];
      if (u == v) continue;
      g->adj[fill[u]++] = v;
      g->adj[fill[v]++] = u;
    }
  free(fill);
#pragma omp parallel for schedule(dynamic, 1024)
  for (int64_t v = 0; v < (int64_t)nv; ++v) {
    uint32_t* a = g->adj + g->start[v];
    const uint64_t n = g->start[v + 1] - g->start[v];
    qsort(a, n, 4, cmp_u32);
    uint64_t k = 0;
    for (uint64_t i = 0; i < n; ++i)
      if (k == 0 || a[i] != a[k - 1]) a[k++] = a[i];
    g->deg[v] = (uint32_t)k;
  }
  return 0;
}

// Batagelj-Zaversnik: core[v] for every v
static int bz(uint32_t nv, const Graph* g, uint32_t* core) {
  uint32_t md = 0;
  for (uint32_t v = 0; v < nv; ++v) md = g->deg[v] > md ? g->deg[v] : md;
  uint32_t* bin = calloc((size_t)md + 2, 4);
  uint32_t* pos = malloc((size_t)nv * 4 + 4);
  uint32_t* vert = malloc((size_t)nv * 4 + 4);
  if (!bin || !pos || !vert) { free(bin); free(pos); free(vert); return -2; }
  for (uint32_t v = 0; v < nv; ++v) { core[v] = g->deg[v]; bin[core[v]]++; }
  uint32_t at = 0;
  for (uint32_t d = 0; d <= md; ++d) { const uint32_t n = bin[d]; bin[d] = at; at += n; }
  for (uint32_t v = 0; v < nv; ++v) { pos[v] = bin[core[v]]; vert[pos[v]] = v; bin[core[v]]++; }
  for (uint32_t d = md; d > 0; --d) bin[d] = bin[d - 1];
  bin[0] = 0;
  for (uint32_t i = 0; i < nv; ++i) {
    const uint32_t v = vert[i];
    for (uint64_t e = g->start[v]; e < g->start[v] + g->deg[v]; ++e) {
      const uint32_t u = g->adj[e];
      if (core[u] > core[v]) {  // move u to the front of its bin, then into the bin below
        const uint32_t du = core[u], pu = pos[u], pw = bin[du], w = vert[pw];
        if (u != w) { pos[u] = pw; vert[pu] = w; pos[w] = pu; vert[pw] = u; }
        bin[du]++;
        core[u]--;
      }
    }
  }
  free(bin);
  free(pos);
  free(vert);
  return 0;
}

// the level-synchronous schedule; stats[1] = rounds, [2] = levels, [3] = degeneracy, [4] = largest |F|
static int sync_peel(uint32_t nv, const Graph* g, uint32_t* core, uint64_t* trace_f, uint32_t* trace_k, uint64_t* stats) {
  uint32_t* deg = malloc((size_t)nv * 4 + 4);
  uint32_t* alive = malloc((size_t)nv * 4 + 4);
  uint32_t* f = malloc((size_t)nv * 4 + 4);
  uint32_t* next = malloc((size_t)nv * 4 + 4);
  if (!deg || !alive || !f || !next) { free(deg); free(alive); free(f); free(next); return -2; }
  const uint32_t unset = 0xFFFFFFFFu;
  for (uint32_t v = 0; v < nv; ++v) { deg[v] = g->deg[v]; core[v] = unset; alive[v] = v; }
  uint32_t n_alive = nv, k = 0;
  uint64_t rounds = 0, levels = 0, widest = 0;
  while (n_alive) {
    uint32_t n = 0, least = unset;
    for (uint32_t i = 0; i < n_alive; ++i)
      if (core[alive[i]] == unset) {
        alive[n++] = alive[i];
        least = deg[alive[i]] < least ? deg[alive[i]] : least;
      }
    n_alive = n;
    if (!n_alive) break;
    k = least > k ? least : k;
    uint32_t nf = 0;
    for (uint32_t i = 0; i < n_alive; ++i)
      if (deg[alive[i]] <= k) f[nf++] = alive[i];
    levels++;
    while (nf) {
      trace_f[rounds] = nf;
      trace_k[rounds] = k;
      rounds++;
      widest = nf > widest ? nf : widest;
      for (uint32_t i = 0; i < nf; ++i) core[f[i]] = k;
      uint32_t nn = 0;
      for (uint32_t i = 0; i < nf; ++i) {
        const uint32_t v = f[i];
        for (uint64_t e = g->start[v]; e < g->start[v] + g->deg[v]; ++e) {
          const uint32_t u = g->adj[e];
          if (core[u] == unset && --deg[u] == k) next[nn++] = u;
        }
      }
      uint32_t* t = f;
      f = next;
      next = t;
      nf = nn;
    }
  }
  stats[1] = rounds;
  stats[2] = levels;
  stats[3] = k;
  stats[4] = widest;
  free(deg);
  free(alive);
  free(f);
  free(next);
  return 0;
}

// stats[0] = m (undirected simple edges), [1] = rounds, [2] = levels, [3] = degeneracy, [4] = largest |F|.  trace_f /
// trace_k hold at least nv entries.  Returns 0, -1 when a source id is >= nv, -2 when out of memory.
int kco_run(uint32_t nv, const uint64_t* row_end, const uint32_t* src, uint32_t* core_bz, uint32_t* core_sync, uint64_t* trace_f,
            uint32_t* trace_k, uint64_t* stats) {
  Graph g;
  int rc = graph_build(nv, row_end, src, &g);
  if (rc == 0) {
    uint64_t twice = 0;
    for (uint32_t v = 0; v < nv; ++v) twice += g.deg[v];
    stats[0] = twice / 2;
    rc = bz(nv, &g, core_bz);
  }
  if (rc == 0) rc = sync_peel(nv, &g, core_sync, trace_f, trace_k, stats);
  graph_free(&g);
  return rc;
}

// bad[v] = 1 iff v is not a fixpoint of the h-index operator under `core`: with c = core[v], a = |{u in N(v) :
// core[u] >= c}| and b = |{u in N(v) : core[u] >= c + 1}|, a < c or b >= c + 1.  Returns the count, or -1 / -2 as above.
int64_t kco_check(uint32_t nv, const uint64_t* row_end, const uint32_t* src, const uint32_t* core, uint8_t* bad) {
  Graph g;
  const int rc = graph_build(nv, row_end, src, &g);
  if (rc) { graph_free(&g); return rc; }
  int64_t total = 0;
#pragma omp parallel for schedule(dynamic, 1024) reduction(+ : total)
  for (int64_t v = 0; v < (int64_t)nv; ++v) {
    const uint64_t c = core[v];
    uint64_t a = 0, b = 0;
    for (uint64_t e = g.start[v]; e < g.start[v] + g.deg[v]; ++e) {
      const uint64_t cu = core[g.adj[e]];
      a += cu >= c;
      b += cu >= c + 1;
    }
    bad[v] = a < c || b >= c + 1;
    total += bad[v];
  }
  graph_free(&g);
  return total;
}
