"""App drivers — the iteration loops of the reference's four top_level_tasks, on top of the C ABI.

pagerank   : pagerank/pagerank.cc:105-118     (-ni fixed iterations)
components : components/components.cc:108-135 (run until no partition reports an active vertex)
sssp       : sssp/sssp.cc                     (same loop, -start; with weights: weighted SSSP, ours)
colfilter  : col_filter/colfilter.cc:71-81    (-ni fixed iterations)
betweenness: Brandes from a list of sources over the SSSP engine's hop levels, or with weights over the weighted
             SSSP distances (ours; the reference has no BC)
triangles  : exact triangle counts of the undirected simple graph (ours)
core_number: exact core numbers of the undirected simple graph, by level-synchronous peeling (ours)
truss      : exact edge support and truss numbers of the undirected simple graph, by level-synchronous edge peeling (ours)
Single-rank convenience wrappers; multi-GPU callers drive LuxGraph directly (see bench.py).
"""
import numpy as np

from .binding import LuxGraph, APP_PAGERANK, APP_CC, APP_SSSP, APP_COLFILTER, APP_SSSP_WEIGHTED, APP_BC, APP_BC_WEIGHTED, APP_TC, APP_KCORE, APP_TRUSS


def pagerank(row_end, src, num_iter=10, device=0):
    """Returns the array the reference holds in dist_lr[ni % 2]: rank / out-degree (pagerank_gpu.cu:98-100)."""
    with LuxGraph.from_csc(row_end, src, app=APP_PAGERANK, device=device) as g:
        g.init()
        g.iterate(num_iter)
        return g.values()


def components(row_end, src, device=0, check=False):
    with LuxGraph.from_csc(row_end, src, app=APP_CC, device=device) as g:
        g.init()
        iters = g.run_to_convergence()
        out = dict(labels=g.values(), iters=iters, trace=g.trace())
        if check:
            out["mistakes"] = g.check()
        return out


def sssp(row_end, src, start=0, device=0, check=False, weight=None):
    """Hop counts (INF = nv), or with `weight` (i32 per edge, CSC order, >= 0) weighted shortest-path distances
    (INF = DIST_INF = 2^32 - 1, sums saturate at INF)."""
    app = APP_SSSP if weight is None else APP_SSSP_WEIGHTED
    with LuxGraph.from_csc(row_end, src, weight, app=app, start=start, device=device) as g:
        g.init()
        iters = g.run_to_convergence()
        out = dict(labels=g.values(), iters=iters, trace=g.trace())
        if check:
            out["mistakes"] = g.check()
        return out


def colfilter(row_end, src, weight, num_iter=10, device=0):
    with LuxGraph.from_csc(row_end, src, weight, app=APP_COLFILTER, device=device) as g:
        g.init()
        g.iterate(num_iter)
        return g.values()


def betweenness(row_end, src, sources=None, device=0, weight=None):
    """Betweenness centrality scores (f64 [nv], not normalised) over the CSC's directed edges: the sum over the sources
    s != v of Brandes' dependency delta_s(v).  Unweighted paths, or with `weight` (i32 per edge, CSC order, every weight
    >= 1) shortest paths by weighted distance, where only the edges on a shortest path count.  sources=None means every
    vertex (exact BC); a sample gives the usual estimate, a source listed twice counts twice."""
    nv = len(row_end)
    srcs = np.arange(nv, dtype=np.uint32) if sources is None else np.asarray(sources)
    app = APP_BC if weight is None else APP_BC_WEIGHTED
    with LuxGraph.from_csc(row_end, src, weight, app=app, device=device) as g:
        g.init()
        g.bc_run(srcs)
        return g.values()


def triangles(row_end, src, device=0):
    """Triangle counts of the CSC read as an undirected simple graph ({u, v} is an edge iff u != v and u -> v or v -> u is
    stored; weights are ignored): dict(total = number of triangles, per_vertex = u64 [nv] triangles containing each
    vertex)."""
    with LuxGraph.from_csc(row_end, src, app=APP_TC, device=device) as g:
        g.init()
        total = g.tc_run()
        return dict(total=total, per_vertex=g.values())


def core_number(row_end, src, device=0):
    """Core numbers of the CSC read as an undirected simple graph ({u, v} is an edge iff u != v and u -> v or v -> u is
    stored; weights are ignored), as networkx's core_number(): dict(core = u32 [nv], degeneracy = the largest core
    number, rounds = the peel's rounds)."""
    with LuxGraph.from_csc(row_end, src, app=APP_KCORE, device=device) as g:
        g.init()
        degeneracy = g.kcore_run()
        return dict(core=g.values(), degeneracy=degeneracy, rounds=g.stats()["iterations"])


def truss(row_end, src, device=0):
    """k-truss decomposition of the CSC read as an undirected simple graph ({u, v} is an edge iff u != v and u -> v or
    v -> u is stored; weights are ignored): dict(lo, hi = u32 [m] the edges in ascending (lo, hi) order, support = u32 [m]
    triangles at each edge, truss = u32 [m] truss numbers (the edges with truss >= k are networkx's k_truss(G, k)),
    vertex = u32 [nv] the largest truss number at each vertex, kmax, rounds = the peel's rounds)."""
    with LuxGraph.from_csc(row_end, src, app=APP_TRUSS, device=device) as g:
        g.init()
        kmax = g.truss_run()
        lo, hi, support, tr = g.truss_edges()
        return dict(lo=lo, hi=hi, support=support, truss=tr, vertex=g.values(), kmax=kmax, rounds=g.stats()["iterations"])
