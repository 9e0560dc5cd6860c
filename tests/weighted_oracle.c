/*
 * weighted_oracle.c — CPU oracle of weighted SSSP (test infrastructure, NOT product code; the product never links it).
 *
 * The reference has no weighted SSSP (its "SSSP" is a hop count, sssp_gpu.cu:122), so nothing can be replayed: this
 * restates the semantics of LUXB_SSSP_WEIGHTED (include/lux_b200.h) in plain C + OpenMP, with the iteration structure
 * of the hop-count oracle (oracle/lux_oracle.c lo_label_run: Jacobi iterations, pull when the global active count
 * > nv/16, per-partition frontier representation rules, halt on zero active).  It is pinned by an independent
 * algorithm: tests/test_sssp_weighted_oracle.py compares its labels with scipy's Dijkstra.
 *   D[start] = 0, every other vertex INF = 2^32 - 1;  cand = sat_add(D[u], w) = min(D[u] + w, INF), no wrap-around.
 * Weights are i32 in CSC edge order, >= 0.  The partition bounds come from the caller (oracle.partition).
 */
#include <stdint.h>
#include <stdlib.h>
#include <string.h>
#ifdef _OPENMP
#include <omp.h>
#endif

typedef uint32_t V_ID;
typedef uint64_t E_ID;

#define WO_INF 0xFFFFFFFFu
#define WO_SPARSE_THRESHOLD 16      /* components/app.h:19 */
#define WO_DENSE_BITMAP 0x1234567u  /* core/graph.h:102 */
#define WO_SPARSE_QUEUE 0x7654321u  /* core/graph.h:103 */

static inline uint64_t splitmix64(uint64_t x) {
  uint64_t z = x + 0x9E3779B97F4A7C15ull;
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  return z ^ (z >> 31);
}

/* directed RMAT weight in [1, 255] of src -> dst; lux_b200/csrc/build.cuh rmat_weight must match it bit for bit */
int32_t wo_rmat_weight(uint64_t seed, V_ID src, V_ID dst) {
  uint64_t h = splitmix64(splitmix64(seed ^ 0x9E3779B97F4A7C15ull) ^ (((uint64_t)dst << 32) | src));
  return (int32_t)(1 + (h >> 32) % 255);
}

void wo_rmat_csc_weights(uint64_t seed, V_ID nv, const E_ID* row_end, const V_ID* src, int32_t* weight) {
#pragma omp parallel for schedule(dynamic, 4096)
  for (int64_t vv = 0; vv < (int64_t)nv; vv++) {
    V_ID v = (V_ID)vv;
    for (E_ID k = (v == 0 ? 0 : row_end[v - 1]); k < row_end[v]; k++) weight[k] = wo_rmat_weight(seed, src[k], v);
  }
}

static inline V_ID sat_add(V_ID d, int32_t w) {
  uint64_t s = (uint64_t)d + (uint32_t)w;
  return s < WO_INF ? (V_ID)s : WO_INF;
}
uint32_t wo_sat_add(uint32_t d, int32_t w) { return sat_add(d, w); }

void wo_init(V_ID nv, V_ID start, V_ID* label) {
  for (V_ID v = 0; v < nv; v++) label[v] = WO_INF;
  if (start < nv) label[start] = 0;
}

/* Jacobi pull sweep over [v_lo, v_hi]; returns #vertices whose distance changed */
uint64_t wo_pull_range(const E_ID* row_end, const V_ID* src, const int32_t* w, const V_ID* old_l, V_ID* new_l, V_ID v_lo,
                       V_ID v_hi) {
  uint64_t changed = 0;
#pragma omp parallel for schedule(dynamic, 4096) reduction(+ : changed)
  for (int64_t vv = v_lo; vv <= (int64_t)v_hi; vv++) {
    V_ID v = (V_ID)vv;
    V_ID cur = old_l[v];
    for (E_ID k = (v == 0 ? 0 : row_end[v - 1]); k < row_end[v]; k++) {
      V_ID c = sat_add(old_l[src[k]], w[k]);
      if (c < cur) cur = c;
    }
    new_l[v] = cur;
    changed += cur != old_l[v];
  }
  return changed;
}

/* CSR-by-source over the edges of destinations [v_lo, v_hi], ascending edge index inside a source (the order of
 * oracle lo_build_push_csr), with each edge's weight carried to out_w[] aligned with out_dst[] */
void wo_build_push_csr(V_ID nv, const E_ID* row_end, const V_ID* src, const int32_t* w, V_ID v_lo, V_ID v_hi, E_ID* out_end,
                       V_ID* out_dst, int32_t* out_w) {
  E_ID e_lo = v_lo == 0 ? 0 : row_end[v_lo - 1], e_hi = row_end[v_hi];
  E_ID* cursor = (E_ID*)calloc((size_t)nv + 1, sizeof(E_ID));
  for (E_ID e = e_lo; e < e_hi; e++) cursor[src[e] + 1]++;
  for (V_ID u = 0; u < nv; u++) cursor[u + 1] += cursor[u];
  for (V_ID u = 0; u < nv; u++) out_end[u] = cursor[u + 1];
  for (V_ID v = v_lo; v <= v_hi; v++)
    for (E_ID e = (v == 0 ? 0 : row_end[v - 1]); e < row_end[v]; e++) {
      E_ID pos = cursor[src[e]]++;
      out_dst[pos] = v;
      out_w[pos] = w[e];
    }
  free(cursor);
}

/* Whole-graph run over P partitions [rl[p], rr[p]] (empty: rr < rl).  Records per iteration the global active count,
 * the direction (1 = pull) and each partition's frontier type; returns the number of iterations including the final
 * all-zero one. */
int wo_run(V_ID nv, E_ID ne, const E_ID* row_end, const V_ID* src, const int32_t* w, int P, const V_ID* rl, const V_ID* rr,
           V_ID start, V_ID* label_out, int max_iters, uint64_t* active_per_iter, int* pull_per_iter, uint32_t* type_per_iter_part) {
  V_ID* old_l = malloc(sizeof(V_ID) * (size_t)nv);
  V_ID* new_l = malloc(sizeof(V_ID) * (size_t)nv);
  uint8_t* active = calloc(nv, 1);
  uint32_t* ftype = malloc(sizeof(uint32_t) * P);
  uint64_t* fcount = malloc(sizeof(uint64_t) * P);
  wo_init(nv, start, new_l);
  for (int p = 0; p < P; p++) {  /* initial frontier {start}, sparse */
    ftype[p] = WO_SPARSE_QUEUE;
    fcount[p] = (rr[p] >= rl[p] && start >= rl[p] && start <= rr[p]) ? 1 : 0;
  }
  if (start < nv) active[start] = 1;
  E_ID* out_end = malloc(sizeof(E_ID) * (size_t)nv);
  V_ID* out_dst = malloc(sizeof(V_ID) * (size_t)(ne ? ne : 1));
  int32_t* out_w = malloc(sizeof(int32_t) * (size_t)(ne ? ne : 1));
  wo_build_push_csr(nv, row_end, src, w, 0, nv - 1, out_end, out_dst, out_w);
  int it = 0;
  for (; it < max_iters; it++) {
    memcpy(old_l, new_l, sizeof(V_ID) * (size_t)nv);
    uint64_t old_size = 0;
    int dense_parts = 0, sparse_parts = 0;
    for (int p = 0; p < P; p++) {
      old_size += fcount[p];
      if (ftype[p] == WO_DENSE_BITMAP) dense_parts++; else sparse_parts++;
    }
    int dense_fq = dense_parts >= sparse_parts;
    int pull = old_size > (uint64_t)(nv / 16);
    if (pull) {
      dense_fq = 1;
      wo_pull_range(row_end, src, w, old_l, new_l, 0, nv - 1);
    } else {
      for (V_ID u = 0; u < nv; u++) {
        if (!active[u]) continue;
        for (E_ID k = (u == 0 ? 0 : out_end[u - 1]); k < out_end[u]; k++) {
          V_ID c = sat_add(old_l[u], out_w[k]);
          if (c < new_l[out_dst[k]]) new_l[out_dst[k]] = c;
        }
      }
    }
    uint64_t total = 0;
    for (int p = 0; p < P; p++) {
      uint64_t c = 0;
      if (rr[p] >= rl[p])
        for (V_ID v = rl[p]; v <= rr[p]; v++) { active[v] = old_l[v] != new_l[v]; c += active[v]; }
      uint64_t max_nodes = (uint64_t)((rr[p] >= rl[p] ? rr[p] - rl[p] : 0) / WO_SPARSE_THRESHOLD + 100);
      int d = dense_fq;
      if (d) { if (c < max_nodes) d = 0; }
      else { if (c >= max_nodes) d = 1; }
      ftype[p] = d ? WO_DENSE_BITMAP : WO_SPARSE_QUEUE;
      fcount[p] = c;
      total += c;
      if (type_per_iter_part) type_per_iter_part[(size_t)it * P + p] = ftype[p];
    }
    if (active_per_iter) active_per_iter[it] = total;
    if (pull_per_iter) pull_per_iter[it] = pull;
    if (total == 0) { it++; break; }
  }
  memcpy(label_out, new_l, sizeof(V_ID) * (size_t)nv);
  free(old_l); free(new_l); free(active); free(ftype); free(fcount); free(out_end); free(out_dst); free(out_w);
  return it;
}

/* check: in-edges with D[u] != INF && D[v] > sat_add(D[u], w) */
uint64_t wo_check(V_ID nv, const E_ID* row_end, const V_ID* src, const int32_t* w, const V_ID* label) {
  uint64_t bad = 0;
#pragma omp parallel for schedule(dynamic, 4096) reduction(+ : bad)
  for (int64_t vv = 0; vv < (int64_t)nv; vv++) {
    V_ID v = (V_ID)vv;
    for (E_ID k = (v == 0 ? 0 : row_end[v - 1]); k < row_end[v]; k++) {
      V_ID lu = label[src[k]];
      bad += (lu != WO_INF) && (label[v] > sat_add(lu, w[k]));
    }
  }
  return bad;
}
