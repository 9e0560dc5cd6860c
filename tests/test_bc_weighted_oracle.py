"""The weighted betweenness-centrality oracle (tests/bc_weighted_oracle.c) against independent answers, on the CPU:
networkx's weighted Brandes (on graphs reduced to the lightest of each set of parallel edges, since networkx collapses
them), scipy's Dijkstra and the weighted SSSP oracle for the distances, the unweighted BC oracle bit for bit under unit
weights, hand-worked graphs, and the exact weighted forest generator's own promises."""
import numpy as np
import pytest

import oracle as O
import bc_oracle as B
import bc_weighted_oracle as W
import weighted_oracle as WO
from graphs import ALL_SMALL, rmat

nx = pytest.importorskip("networkx")


def lightest(row_end, src, weight):
    """One edge per (u, v), of the smallest weight: what networkx sees of a multigraph."""
    dst = W.csc_dst(row_end)
    if len(src) == 0:
        return row_end, src, weight
    order = np.lexsort((weight, src, dst))
    s, d, w = src.astype(np.int64)[order], dst[order], weight[order]
    first = np.concatenate([[True], (s[1:] != s[:-1]) | (d[1:] != d[:-1])])
    return W.edges_to_csc(len(row_end), s[first], d[first], w[first])


def nx_graph(row_end, src, weight):
    G = nx.DiGraph()
    G.add_nodes_from(range(len(row_end)))
    G.add_weighted_edges_from(zip(src.tolist(), W.csc_dst(row_end).tolist(), weight.tolist()))
    return G


def nx_scores(row_end, src, weight, sources=None):
    G = nx_graph(row_end, src, weight)
    if sources is None:
        d = nx.betweenness_centrality(G, weight="weight", normalized=False)
    else:
        d = nx.betweenness_centrality_subset(G, sources=[int(s) for s in sources], targets=list(G.nodes), normalized=False,
                                             weight="weight")
    return np.array([d[v] for v in range(len(row_end))], np.float64)


def sample(nv, k, seed):
    return np.random.default_rng(seed).choice(nv, min(k, nv), replace=False).astype(np.uint32)


def close(a, b, rtol=1e-12):
    np.testing.assert_allclose(a, b, rtol=rtol, atol=1e-9)


def weights(kind, ne, seed=7):
    rng = np.random.default_rng(seed)
    return (rng.integers(1, 256, ne) if kind == "w255" else rng.integers(1, 3, ne)).astype(np.int32)


@pytest.mark.parametrize("kind", ["w255", "w12"])
@pytest.mark.parametrize("name", sorted(ALL_SMALL))
def test_networkx_small_fixtures(name, kind):
    row_end, src = ALL_SMALL[name]()
    row_end, src, w = lightest(row_end, src, weights(kind, len(src)))
    nv, ne = len(row_end), len(src)
    if nv * max(ne, 1) <= 2e7:
        close(W.scores(row_end, src, w), nx_scores(row_end, src, w))
    S = sample(nv, 48, 5)
    close(W.scores(row_end, src, w, S), nx_scores(row_end, src, w, S))


@pytest.mark.parametrize("scale", [10, 12])
def test_networkx_rmat_generator_weights(scale):
    row_end, src = rmat(scale)
    row_end, src, w = lightest(row_end, src, WO.rmat_weights(27, row_end, src))
    S = sample(len(row_end), 64 if scale == 12 else 1024, scale)
    close(W.scores(row_end, src, w, S), nx_scores(row_end, src, w, S))


@pytest.mark.parametrize("name", ["rmat10", "hand5", "two_components", "trailing_isolated", "star"])
def test_distances_equal_weighted_sssp_and_dijkstra(name):
    from scipy.sparse import csr_matrix
    from scipy.sparse.csgraph import dijkstra
    row_end, src = ALL_SMALL[name]()
    nv = len(row_end)
    w = weights("w255", len(src))
    lo = lightest(row_end, src, w)  # scipy keeps one entry per (u, v) as well
    A = csr_matrix((lo[2].astype(np.float64), (lo[1].astype(np.int64), W.csc_dst(lo[0]))), shape=(nv, nv))
    for s in (0, nv // 3, nv - 1):
        dist, sigma, delta = W.source_state(row_end, src, w, s)
        assert np.array_equal(dist, WO.label_run(row_end, src, w, start=s)["labels"])
        ref = dijkstra(A, indices=s)
        assert np.array_equal(dist == W.INF, np.isinf(ref))
        assert np.array_equal(dist[dist != W.INF].astype(np.float64), ref[~np.isinf(ref)])
        assert np.all(sigma == np.floor(sigma)) and np.all((sigma > 0) == (dist != W.INF))
        assert np.all(delta[dist == W.INF] == 0) and np.all(delta >= 0)


@pytest.mark.parametrize("name", sorted(ALL_SMALL))
def test_unit_weights_are_unweighted_bc_bit_for_bit(name):
    row_end, src = ALL_SMALL[name]()
    nv = len(row_end)
    S = sample(nv, 64, 3)
    a = W.run(row_end, src, np.ones(len(src), np.int32), S)
    b = B.run(row_end, src, S)
    for k in ("scores", "sigma", "delta"):
        assert np.array_equal(a[k], b[k]), k
    assert np.array_equal(np.where(a["dist"] == W.INF, nv, a["dist"]), b["lev"])
    assert np.array_equal(a["classes"], b["levels"])


def diamond(w3, double=None):
    """0 -> 1 -> 3 and 0 -> 2 -> 3 (weights 1, 2 and 2, w3), then 3 -> 4; `double` appends another 0 -> 1 of that weight."""
    s, d, w = [0, 0, 1, 2, 3], [1, 2, 3, 3, 4], [1, 2, 2, w3, 1]
    if double is not None:
        s, d, w = s + [0], d + [1], w + [double]
    return W.edges_to_csc(5, s, d, w)


def test_weighted_diamond_longer_branch_and_tie():
    # 0 -> 2 -> 3 costs 2 + 2 = 4 against 0 -> 1 -> 3 at 3: one shortest path, through 1 only
    r = W.run(*diamond(2), [0])
    assert r["dist"].tolist() == [0, 1, 2, 3, 4] and r["sigma"].tolist() == [1, 1, 1, 1, 1]
    close(W.scores(*diamond(2), [0]), [0, 2, 0, 1, 0])
    # w(2, 3) = 1 ties the two branches: sigma[3] = 2, each middle vertex carries half of the paths to 3 and 4
    r = W.run(*diamond(1), [0])
    assert r["dist"].tolist() == [0, 1, 2, 3, 4] and r["sigma"].tolist() == [1, 1, 1, 2, 2]
    close(r["delta"], [r["delta"][0], 1, 1, 1, 0])
    close(W.scores(*diamond(1)), nx_scores(*diamond(1)))


def test_parallel_edges_count_only_at_the_minimal_weight():
    # a second 0 -> 1 at the same weight doubles sigma[1] and the paths through it; at a larger weight it changes nothing
    r = W.run(*diamond(1, double=1), [0])
    assert r["sigma"].tolist() == [1, 2, 1, 3, 3]
    close(r["delta"], [r["delta"][0], 4 / 3, 2 / 3, 1, 0])
    plain = W.run(*diamond(1), [0])
    heavy = W.run(*diamond(1, double=5), [0])
    for k in ("dist", "sigma", "delta", "scores"):
        assert np.array_equal(heavy[k], plain[k]), k


def test_self_loop_is_never_tight():
    row_end, src = rmat(10)
    nv = len(row_end)
    w = weights("w12", len(src))
    loops = np.arange(0, nv, 3)
    row_end2, src2, w2 = W.edges_to_csc(nv, np.concatenate([src, loops]), np.concatenate([W.csc_dst(row_end), loops]),
                                        np.concatenate([w, np.ones(len(loops), np.int64)]))
    S = sample(nv, 32, 1)
    assert np.array_equal(W.scores(row_end, src, w, S), W.scores(row_end2, src2, w2, S))


def test_isolated_source_contributes_zero():
    row_end, src, w = W.edges_to_csc(6, [0, 1, 1], [1, 2, 3], [3, 1, 7])  # 4 and 5 isolated, 2 and 3 sinks
    for s in (4, 2, 3):
        r = W.run(row_end, src, w, [s])
        assert np.all(r["scores"] == 0) and r["classes"][0] == 1
        assert r["sigma"][s] == 1 and r["sigma"].sum() == 1 and np.all(r["delta"] == 0)
        assert np.all(r["dist"][np.arange(6) != s] == W.INF)
    assert W.scores(row_end, src, w).tolist() == [0, 2, 0, 0, 0, 0]


def test_saturation_chain():
    # 0 -> 1 -> 2 -> 3 with weights 2^31 - 1: D[2] = 2^32 - 2 is reached, D[3] would be past INF and is not
    big = (1 << 31) - 1
    row_end, src, w = W.edges_to_csc(4, [0, 1, 2], [1, 2, 3], [big, big, big])
    r = W.run(row_end, src, w, [0])
    assert r["dist"].tolist() == [0, big, 2 * big, W.INF]
    assert r["sigma"].tolist() == [1, 1, 1, 0] and r["delta"].tolist() == [r["delta"][0], 1, 0, 0]
    assert np.array_equal(r["dist"], WO.label_run(row_end, src, w, start=0)["labels"])
    # a sum that lands exactly on 2^32 - 1 is unreachable too, and its edge is not tight (t of an unreached vertex would
    # divide by sigma = 0)
    row_end, src, w = W.edges_to_csc(4, [0, 1, 2], [1, 2, 3], [big, big, 1])
    r = W.run(row_end, src, w, [0])
    assert r["dist"].tolist() == [0, big, 2 * big, W.INF] and r["delta"].tolist() == [2, 1, 0, 0]
    assert np.all(np.isfinite(r["scores"]))


def test_weights_below_one_are_rejected():
    row_end, src, w = W.edges_to_csc(3, [0, 1], [1, 2], [1, 0])
    with pytest.raises(ValueError, match="w >= 1"):
        W.run(row_end, src, w, [0])
    with pytest.raises(ValueError, match="w >= 1"):
        W.run(row_end, src, np.array([1, -4], np.int32), [0])
    with pytest.raises(ValueError):
        W.run(row_end, src, np.array([1, 1], np.int32), [3])


def forest_checks(f):
    row_end, src, w, roots = f["row_end"], f["src"], f["weight"], f["roots"]
    nv = len(row_end)
    dist_all = np.full(nv, W.INF, np.int64)
    for s in roots:
        dist, sigma, delta = W.source_state(row_end, src, w, s)
        mine = f["tree"] == f["tree"][s]
        assert np.array_equal(dist[mine].astype(np.int64), f["dist"][mine]) and np.all(dist[~mine] == W.INF)
        assert np.array_equal(sigma[mine], np.ldexp(1.0, f["log_sigma"][mine]))  # powers of two
        assert np.array_equal(delta[mine], f["descendants"][mine])               # integers
        dist_all[mine] = dist[mine]
    assert np.array_equal(W.scores(row_end, src, w, roots), f["scores"])
    # the tight edges are exactly the tree edges: one parent per non-root vertex; every other edge misses, some by one
    du, dv = dist_all[src.astype(np.int64)], dist_all[W.csc_dst(row_end)]
    tight = du + w == dv
    assert np.all(tight | (du + w > dv))
    parents = np.unique(np.stack([src[tight].astype(np.int64), W.csc_dst(row_end)[tight]], 1), axis=0)
    counts = np.bincount(parents[:, 1], minlength=nv)
    reached = dist_all != W.INF
    assert np.all(counts[reached & (dist_all > 0)] == 1) and np.all(counts[dist_all == 0] == 0)
    assert np.any(du + w == dv + 1)                                   # near misses
    assert np.any(~tight & (dv > du))                                 # non-tight edges to larger distances
    assert w.min() >= 1 and w[tight].max() <= 255
    return dist_all


def test_small_forest_is_exact():
    forest_checks(W.small_forest())


def test_forest_is_exact_and_has_the_split_cases():
    f = W.forest()
    dist = forest_checks(f)
    row_end = f["row_end"]
    indeg = np.diff(np.concatenate([[0], row_end]).astype(np.int64))
    outdeg = np.bincount(f["src"].astype(np.int64), minlength=len(row_end))
    assert outdeg.max() >= 1 << 17          # a hub whose delta sum is cut into segments
    assert indeg.max() >= 1 << 20           # a vertex whose sigma sum is cut into segments (none of them tight)
    classes = W.run(f["row_end"], f["src"], f["weight"], f["roots"])["classes"]
    assert classes.max() >= 1000            # a chain with at least 1000 distinct distances
    assert len(np.unique(dist[dist != W.INF])) >= 1000
