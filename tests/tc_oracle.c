// tc_oracle.c — CPU oracle of triangle counting (LUXB_TC), test infrastructure only.  C + OpenMP.
//
// Semantics (as in include/lux_b200.h and DESIGN §0): the CSC's directed edges are read as an undirected simple graph,
// {u, v} is an edge iff u != v and u -> v or v -> u is stored (parallel edges, both directions and self-loops collapse,
// weights are ignored).  t[v] = number of triangles containing v (u64), T = sum of t / 3.
//
// Formulation, independent of the device path (no global key sort, no shared-memory counters): the undirected
// neighbour lists are built by a counting sort over the endpoints, then sorted and deduplicated per vertex.  Each edge
// is oriented from the lower to the higher (degree, id); for every u the thread marks N+(u) in a dense per-thread marker
// array, and each w of N+(v), v in N+(u), that carries u's mark closes the triangle {u, v, w}.  Counts go to
// thread-local arrays that are summed at the end.
#include <omp.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

static int cmp_u32(const void* a, const void* b) {
  const uint32_t x = *(const uint32_t*)a, y = *(const uint32_t*)b;
  return (x > y) - (x < y);
}

// stats[0] = T, [1] = m (undirected simple edges), [2] = probes (sum over oriented (u, v) of |N+(v)|),
// [3] = largest |N+(u)|, [4] = threads used.  Returns 0, -1 when a source id is >= nv, -2 when out of memory.
int tco_run(uint32_t nv, uint64_t ne, const uint64_t* row_end, const uint32_t* src, uint64_t* t, uint64_t* stats) {
  (void)ne;
  int rc = -2;
  uint64_t* start = calloc((size_t)nv + 1, 8);
  uint64_t* fill = NULL;
  uint32_t* adj = NULL;
  uint32_t* deg = calloc((size_t)nv + 1, 4);
  uint64_t* ostart = calloc((size_t)nv + 1, 8);
  uint32_t* out = NULL;
  uint64_t* local = NULL;
  uint32_t* mark = NULL;
  if (!start || !deg || !ostart) goto done;
  for (uint32_t v = 0; v < nv; ++v)
    for (uint64_t e = v ? row_end[v - 1] : 0; e < row_end[v]; ++e) {
      const uint32_t u = src[e];
      if (u >= nv) { rc = -1; goto done; }
      if (u == v) continue;
      start[u + 1]++;
      start[v + 1]++;
    }
  for (uint32_t v = 0; v < nv; ++v) start[v + 1] += start[v];
  adj = malloc((size_t)start[nv] * 4 + 4);
  fill = malloc((size_t)nv * 8 + 8);
  if (!adj || !fill) goto done;
  memcpy(fill, start, (size_t)nv * 8);
  for (uint32_t v = 0; v < nv; ++v)
    for (uint64_t e = v ? row_end[v - 1] : 0; e < row_end[v]; ++e) {
      const uint32_t u = src[e];
      if (u == v) continue;
      adj[fill[u]++] = v;
      adj[fill[v]++] = u;
    }
  // sorted, distinct neighbour lists: deg[v] entries from start[v]
#pragma omp parallel for schedule(dynamic, 1024)
  for (int64_t v = 0; v < (int64_t)nv; ++v) {
    uint32_t* a = adj + start[v];
    const uint64_t n = start[v + 1] - start[v];
    qsort(a, n, 4, cmp_u32);
    uint64_t k = 0;
    for (uint64_t i = 0; i < n; ++i)
      if (k == 0 || a[k - 1] != a[i]) a[k++] = a[i];
    deg[v] = (uint32_t)k;
  }
  uint64_t m2 = 0;
  for (uint32_t v = 0; v < nv; ++v) m2 += deg[v];
  // N+(u): the neighbours ranked above u, ascending ids
  for (uint32_t u = 0; u < nv; ++u) {
    uint64_t c = 0;
    for (uint64_t i = 0; i < deg[u]; ++i) {
      const uint32_t v = adj[start[u] + i];
      c += deg[u] < deg[v] || (deg[u] == deg[v] && u < v);
    }
    ostart[u + 1] = ostart[u] + c;
  }
  out = malloc((size_t)ostart[nv] * 4 + 4);
  if (!out) goto done;
  uint64_t max_out = 0;
  for (uint32_t u = 0; u < nv; ++u) {
    uint64_t k = ostart[u];
    for (uint64_t i = 0; i < deg[u]; ++i) {
      const uint32_t v = adj[start[u] + i];
      if (deg[u] < deg[v] || (deg[u] == deg[v] && u < v)) out[k++] = v;
    }
    if (ostart[u + 1] - ostart[u] > max_out) max_out = ostart[u + 1] - ostart[u];
  }
  free(adj);
  adj = NULL;
  // per-thread state: a marker array and a count array of nv entries each, at most ~2 GiB of counts in all
  int nth = omp_get_max_threads();
  const uint64_t cap = (2ull << 30) / ((uint64_t)nv * 8 + 8);
  if ((uint64_t)nth > cap) nth = cap ? (int)cap : 1;
  local = calloc((size_t)nth * nv + 1, 8);
  mark = calloc((size_t)nth * nv + 1, 4);
  if (!local || !mark) goto done;
  uint64_t probes = 0;
#pragma omp parallel num_threads(nth) reduction(+ : probes)
  {
    const int me = omp_get_thread_num();
    uint64_t* cnt = local + (size_t)me * nv;
    uint32_t* mk = mark + (size_t)me * nv;
#pragma omp for schedule(dynamic, 256)
    for (int64_t u = 0; u < (int64_t)nv; ++u) {
      const uint32_t stamp = (uint32_t)u + 1;
      for (uint64_t i = ostart[u]; i < ostart[u + 1]; ++i) mk[out[i]] = stamp;
      uint64_t cu = 0;
      for (uint64_t i = ostart[u]; i < ostart[u + 1]; ++i) {
        const uint32_t v = out[i];
        uint64_t cv = 0;
        probes += ostart[v + 1] - ostart[v];
        for (uint64_t j = ostart[v]; j < ostart[v + 1]; ++j)
          if (mk[out[j]] == stamp) {
            cnt[out[j]]++;
            ++cv;
          }
        cnt[v] += cv;
        cu += cv;
      }
      cnt[u] += cu;
    }
  }
  uint64_t sum = 0;
#pragma omp parallel for reduction(+ : sum)
  for (int64_t v = 0; v < (int64_t)nv; ++v) {
    uint64_t s = 0;
    for (int k = 0; k < nth; ++k) s += local[(size_t)k * nv + v];
    t[v] = s;
    sum += s;
  }
  stats[0] = sum / 3;
  stats[1] = m2 / 2;
  stats[2] = probes;
  stats[3] = max_out;
  stats[4] = (uint64_t)nth;
  rc = 0;
done:
  free(start);
  free(fill);
  free(adj);
  free(deg);
  free(ostart);
  free(out);
  free(local);
  free(mark);
  return rc;
}
