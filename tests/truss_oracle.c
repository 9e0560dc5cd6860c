// truss_oracle.c — CPU oracle of the k-truss decomposition (LUXB_TRUSS), test infrastructure only.  C + OpenMP.
//
// Semantics (as in include/lux_b200.h and DESIGN §3.4e): the CSC's directed edges are read as an undirected simple
// graph, {u, v} is an edge iff u != v and u -> v or v -> u is stored (parallel edges, both directions and self-loops
// collapse, weights are ignored).  Edge ids are the ranks of (lo, hi), lo < hi, in ascending order.  sup(e) for
// e = {u, v} is |N(u) ∩ N(v)|; τ(e) is the largest k >= 2 such that e lies in a subgraph in which every edge is in at
// least k - 2 triangles of that subgraph; tv(v) is the largest τ at v (0 without edges); kmax the largest τ.
//
// Three computations over the same neighbour lists (counting sort over the endpoints, then sorted and deduplicated per
// vertex, an edge id beside every entry):
//  - support by sorted-list intersection (each entry of the shorter list looked up in the longer one);
//  - τ by the sequential bucket peel of Wang and Cheng: edges kept sorted by current support in bins, the least one
//    removed with τ = its support + 2, the supports above it of its triangles' other edges lowered by one;
//  - τ_sync and the trace by the level-synchronous schedule of the device, sequentially, with ℓ = k - 2: ℓ = 0; while an
//    edge is alive: ℓ = max(ℓ, min sup over the alive edges); repeat: F = {alive e : sup(e) <= ℓ}, stop if F is empty;
//    τ[F] = ℓ + 2; every triangle whose three edges were alive at the start of the round and which has an edge in F
//    lowers the support of each of its edges not in F by one, applied from the F edge of the smallest id; remove F.
// tro_check counts the edges that fail the truss check (the luxb_check of LUXB_TRUSS).
#include <omp.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

static int cmp_u32(const void* a, const void* b) {
  const uint32_t x = *(const uint32_t*)a, y = *(const uint32_t*)b;
  return (x > y) - (x < y);
}

typedef struct {
  uint32_t nv;
  uint64_t m;
  uint64_t* start;  // [nv + 1] list of v at adj[start[v], start[v] + deg[v])
  uint32_t* deg;    // [nv] distinct neighbours
  uint32_t* adj;    // neighbours, ascending
  uint32_t* eid;    // edge id of every entry
  uint32_t* lo;     // [m] endpoints of every edge
  uint32_t* hi;
} Graph;

static void graph_free(Graph* g) {
  free(g->start);
  free(g->deg);
  free(g->adj);
  free(g->eid);
  free(g->lo);
  free(g->hi);
}

// position of w in v's list, or -1
static int64_t find(const Graph* g, uint32_t v, uint32_t w) {
  uint64_t b = g->start[v], e = g->start[v] + g->deg[v];
  while (b < e) {
    const uint64_t mid = b + (e - b) / 2;
    if (g->adj[mid] < w) b = mid + 1; else e = mid;
  }
  return b < g->start[v] + g->deg[v] && g->adj[b] == w ? (int64_t)b : -1;
}

// 0, -1 when a source id is >= nv, -2 when out of memory, -4 when m >= 2^32
static int graph_build(uint32_t nv, const uint64_t* row_end, const uint32_t* src, Graph* g) {
  memset(g, 0, sizeof(*g));
  g->nv = nv;
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
  g->eid = malloc((size_t)g->start[nv] * 4 + 4);
  uint64_t* fill = malloc((size_t)nv * 8 + 8);
  if (!g->adj || !g->eid || !fill) { free(fill); return -2; }
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
  // edge ids: (lo, hi) ascending = v ascending, then the entries above v in its list
  uint64_t m = 0;
  for (uint32_t v = 0; v < nv; ++v)
    for (uint64_t j = g->start[v]; j < g->start[v] + g->deg[v]; ++j)
      if (g->adj[j] > v) ++m;
  if (m >= (1ull << 32)) return -4;
  g->m = m;
  g->lo = malloc(m * 4 + 4);
  g->hi = malloc(m * 4 + 4);
  if (!g->lo || !g->hi) return -2;
  m = 0;
  for (uint32_t v = 0; v < nv; ++v)
    for (uint64_t j = g->start[v]; j < g->start[v] + g->deg[v]; ++j)
      if (g->adj[j] > v) {
        g->lo[m] = v;
        g->hi[m] = g->adj[j];
        g->eid[j] = (uint32_t)m++;
      }
#pragma omp parallel for schedule(dynamic, 1024)
  for (int64_t v = 0; v < (int64_t)nv; ++v)
    for (uint64_t j = g->start[v]; j < g->start[v] + g->deg[v]; ++j)
      if (g->adj[j] < v) g->eid[j] = g->eid[find(g, g->adj[j], (uint32_t)v)];
  return 0;
}

// the triangles of edge e: for every common neighbour w, the ids of {u, w} and {v, w}
#define FOR_TRIANGLES(g, e, e1, e2, ...)                                                         \
  do {                                                                                           \
    uint32_t a_ = (g)->lo[e], b_ = (g)->hi[e];                                                   \
    if ((g)->deg[b_] < (g)->deg[a_]) { const uint32_t t_ = a_; a_ = b_; b_ = t_; }               \
    for (uint64_t j_ = (g)->start[a_]; j_ < (g)->start[a_] + (g)->deg[a_]; ++j_) {               \
      const int64_t p_ = find((g), b_, (g)->adj[j_]);                                            \
      if (p_ < 0) continue;                                                                      \
      const uint32_t e1 = (g)->eid[j_], e2 = (g)->eid[p_];                                       \
      __VA_ARGS__                                                                                \
    }                                                                                            \
  } while (0)

static void support(const Graph* g, uint32_t* sup) {
#pragma omp parallel for schedule(dynamic, 256)
  for (int64_t e = 0; e < (int64_t)g->m; ++e) {
    uint32_t c = 0;
    FOR_TRIANGLES(g, e, e1, e2, { (void)e1; (void)e2; ++c; });
    sup[e] = c;
  }
}

// Wang-Cheng bucket peel
static int bucket_peel(const Graph* g, const uint32_t* sup0, uint32_t* tau) {
  const uint64_t m = g->m;
  uint32_t ms = 0;
  for (uint64_t e = 0; e < m; ++e) ms = sup0[e] > ms ? sup0[e] : ms;
  uint32_t* s = malloc(m * 4 + 4);
  uint64_t* bin = calloc((size_t)ms + 2, 8);
  uint64_t* pos = malloc(m * 8 + 8);
  uint32_t* vert = malloc(m * 4 + 4);
  uint8_t* gone = calloc(m + 1, 1);
  if (!s || !bin || !pos || !vert || !gone) { free(s); free(bin); free(pos); free(vert); free(gone); return -2; }
  for (uint64_t e = 0; e < m; ++e) { s[e] = sup0[e]; bin[s[e]]++; }
  uint64_t at = 0;
  for (uint32_t d = 0; d <= ms; ++d) { const uint64_t n = bin[d]; bin[d] = at; at += n; }
  for (uint64_t e = 0; e < m; ++e) { pos[e] = bin[s[e]]; vert[pos[e]] = (uint32_t)e; bin[s[e]]++; }
  for (uint32_t d = ms; d > 0; --d) bin[d] = bin[d - 1];
  bin[0] = 0;
  for (uint64_t i = 0; i < m; ++i) {
    const uint32_t e = vert[i];
    tau[e] = s[e] + 2;
    FOR_TRIANGLES(g, e, e1, e2, {
      if (gone[e1] || gone[e2]) continue;
      const uint32_t xs[2] = {e1, e2};
      for (int q = 0; q < 2; ++q) {
        const uint32_t x = xs[q];
        if (s[x] > s[e]) {  // move x to the front of its bin, then into the bin below
          const uint32_t dx = s[x];
          const uint64_t px = pos[x], pw = bin[dx];
          const uint32_t w = vert[pw];
          if (x != w) { pos[x] = pw; vert[px] = w; pos[w] = px; vert[pw] = x; }
          bin[dx]++;
          s[x]--;
        }
      }
    });
    gone[e] = 1;
  }
  free(s);
  free(bin);
  free(pos);
  free(vert);
  free(gone);
  return 0;
}

// the level-synchronous schedule; stats[1] = rounds, [2] = levels, [3] = kmax, [4] = largest |F|.  -3 when a decrement
// finds support 0 (the schedule's invariant broken)
static int sync_peel(const Graph* g, const uint32_t* sup0, uint32_t* tau, uint64_t* trace_f, uint32_t* trace_k, uint64_t* stats) {
  const uint64_t m = g->m;
  uint32_t* s = malloc(m * 4 + 4);
  uint8_t* st = calloc(m + 1, 1);  // 0 alive, 1 in F, 2 removed
  uint32_t* alive = malloc(m * 4 + 4);
  uint32_t* f = malloc(m * 4 + 4);
  uint32_t* next = malloc(m * 4 + 4);
  if (!s || !st || !alive || !f || !next) { free(s); free(st); free(alive); free(f); free(next); return -2; }
  for (uint64_t e = 0; e < m; ++e) { s[e] = sup0[e]; alive[e] = (uint32_t)e; tau[e] = 0; }
  uint64_t n_alive = m, rounds = 0, levels = 0, widest = 0;
  uint32_t l = 0;
  int rc = 0;
  while (n_alive && rc == 0) {
    uint64_t n = 0;
    uint32_t least = 0xFFFFFFFFu;
    for (uint64_t i = 0; i < n_alive; ++i)
      if (st[alive[i]] == 0) {
        alive[n++] = alive[i];
        least = s[alive[i]] < least ? s[alive[i]] : least;
      }
    n_alive = n;
    if (!n_alive) break;
    l = least > l ? least : l;
    uint64_t nf = 0;
    for (uint64_t i = 0; i < n_alive; ++i)
      if (s[alive[i]] <= l) f[nf++] = alive[i];
    levels++;
    while (nf && rc == 0) {
      trace_f[rounds] = nf;
      trace_k[rounds] = l + 2;
      rounds++;
      widest = nf > widest ? nf : widest;
      for (uint64_t i = 0; i < nf; ++i) { st[f[i]] = 1; tau[f[i]] = l + 2; }
      uint64_t nn = 0;
      for (uint64_t i = 0; i < nf; ++i) {
        const uint32_t e = f[i];
        FOR_TRIANGLES(g, e, e1, e2, {
          if (st[e1] == 2 || st[e2] == 2) continue;
          if ((st[e1] == 1 && e1 < e) || (st[e2] == 1 && e2 < e)) continue;
          const uint32_t xs[2] = {e1, e2};
          for (int q = 0; q < 2; ++q) {
            const uint32_t x = xs[q];
            if (st[x] != 0) continue;
            if (s[x] == 0) { rc = -3; continue; }
            if (s[x]-- == l + 1) next[nn++] = x;
          }
        });
      }
      for (uint64_t i = 0; i < nf; ++i) st[f[i]] = 2;
      uint32_t* t = f;
      f = next;
      next = t;
      nf = nn;
    }
  }
  stats[1] = rounds;
  stats[2] = levels;
  stats[3] = rounds ? l + 2 : 0;
  stats[4] = widest;
  free(s);
  free(st);
  free(alive);
  free(f);
  free(next);
  return rc;
}

// m (>= 0) of the undirected simple graph, or -1 / -2 / -4 as graph_build
int64_t tro_num_edges(uint32_t nv, const uint64_t* row_end, const uint32_t* src) {
  Graph g;
  const int rc = graph_build(nv, row_end, src, &g);
  const int64_t m = rc ? rc : (int64_t)g.m;
  graph_free(&g);
  return m;
}

// lo, hi, sup, tau (bucket peel), tau_sync: [m]; tv: [nv] from tau; trace_f / trace_k: at least m entries.  stats[0] = m,
// [1] = rounds, [2] = levels, [3] = kmax (of the schedule), [4] = largest |F|.  Returns 0, or -1 / -2 / -4 as graph_build,
// -3 as sync_peel.
int tro_run(uint32_t nv, const uint64_t* row_end, const uint32_t* src, uint32_t* lo, uint32_t* hi, uint32_t* sup, uint32_t* tau,
            uint32_t* tau_sync, uint32_t* tv, uint64_t* trace_f, uint32_t* trace_k, uint64_t* stats) {
  Graph g;
  int rc = graph_build(nv, row_end, src, &g);
  if (rc == 0) {
    stats[0] = g.m;
    if (g.m) {
      memcpy(lo, g.lo, g.m * 4);
      memcpy(hi, g.hi, g.m * 4);
    }
    support(&g, sup);
    rc = bucket_peel(&g, sup, tau);
  }
  if (rc == 0) {
    memset(tv, 0, (size_t)nv * 4);
    for (uint64_t e = 0; e < g.m; ++e) {
      tv[g.lo[e]] = tau[e] > tv[g.lo[e]] ? tau[e] : tv[g.lo[e]];
      tv[g.hi[e]] = tau[e] > tv[g.hi[e]] ? tau[e] : tv[g.hi[e]];
    }
    rc = sync_peel(&g, sup, tau_sync, trace_f, trace_k, stats);
  }
  graph_free(&g);
  return rc;
}

// bad[e] = 1 iff edge e fails the truss check under `tau` ([m]): with c = tau[e], a = |{w : min(tau(u, w), tau(v, w))
// >= c}| and b the same with >= c + 1 over the common neighbours, c < 2 or a < c - 2 or b >= c - 1.  Returns the count,
// or -1 / -2 / -4 as graph_build.
int64_t tro_check(uint32_t nv, const uint64_t* row_end, const uint32_t* src, const uint32_t* tau, uint8_t* bad) {
  Graph g;
  const int rc = graph_build(nv, row_end, src, &g);
  if (rc) { graph_free(&g); return rc; }
  int64_t total = 0;
#pragma omp parallel for schedule(dynamic, 256) reduction(+ : total)
  for (int64_t e = 0; e < (int64_t)g.m; ++e) {
    const uint64_t c = tau[e];
    uint64_t a = 0, b = 0;
    FOR_TRIANGLES(&g, e, e1, e2, {
      const uint64_t t = tau[e1] < tau[e2] ? tau[e1] : tau[e2];
      a += t >= c;
      b += t >= c + 1;
    });
    bad[e] = c < 2 || a + 2 < c || b + 1 >= c;
    total += bad[e];
  }
  graph_free(&g);
  return total;
}
