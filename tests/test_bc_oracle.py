"""The betweenness-centrality oracle (tests/bc_oracle.c) against independent answers, on the CPU: networkx's Brandes on
de-duplicated graphs (networkx collapses parallel edges), hand-worked graphs (multiplicity included), the hop levels
of the SSSP oracle, and the exact-input forest generator's own promises."""
import numpy as np
import pytest

import oracle as O
import bc_oracle as B
from graphs import ALL_SMALL, rmat, symmetrize, chain, star

nx = pytest.importorskip("networkx")


def dedup(row_end, src):
    nv = len(row_end)
    dst = np.repeat(np.arange(nv, dtype=np.int64), np.diff(np.concatenate([[0], row_end]).astype(np.int64)))
    pairs = np.unique(np.stack([src.astype(np.int64), dst], axis=1), axis=0) if len(src) else np.zeros((0, 2), np.int64)
    return O.edges_to_csc(nv, pairs[:, 0], pairs[:, 1])


def nx_graph(row_end, src):
    nv = len(row_end)
    dst = np.repeat(np.arange(nv, dtype=np.int64), np.diff(np.concatenate([[0], row_end]).astype(np.int64)))
    G = nx.DiGraph()
    G.add_nodes_from(range(nv))
    G.add_edges_from(zip(src.tolist(), dst.tolist()))
    return G


def nx_scores(row_end, src, sources=None):
    G = nx_graph(row_end, src)
    if sources is None:
        d = nx.betweenness_centrality(G, normalized=False)
    else:
        d = nx.betweenness_centrality_subset(G, sources=[int(s) for s in sources], targets=list(G.nodes), normalized=False)
    return np.array([d[v] for v in range(len(row_end))], np.float64)


def sample(nv, k, seed):
    return np.random.default_rng(seed).choice(nv, min(k, nv), replace=False).astype(np.uint32)


def close(a, b, rtol=1e-12):
    np.testing.assert_allclose(a, b, rtol=rtol, atol=1e-9)


@pytest.mark.parametrize("name", sorted(ALL_SMALL))
def test_networkx_small_fixtures(name):
    row_end, src = dedup(*ALL_SMALL[name]())
    nv, ne = len(row_end), len(src)
    if nv * max(ne, 1) <= 2e7:
        close(B.scores(row_end, src), nx_scores(row_end, src))
    S = sample(nv, 48, 5)
    close(B.scores(row_end, src, S), nx_scores(row_end, src, S))


@pytest.mark.parametrize("scale", [10, 12])
def test_networkx_rmat(scale):
    row_end, src = dedup(*rmat(scale))
    S = sample(len(row_end), 64 if scale == 12 else 1024, scale)
    close(B.scores(row_end, src, S), nx_scores(row_end, src, S))


def test_networkx_symmetrised():
    row_end, src = dedup(*symmetrize(*rmat(10)))
    bc = B.scores(row_end, src)
    close(bc, nx_scores(row_end, src))
    # stored with both directions: twice the undirected BC
    G = nx_graph(row_end, src).to_undirected()
    und = nx.betweenness_centrality(G, normalized=False)
    close(bc, 2 * np.array([und[v] for v in range(len(row_end))]))


def test_directed_path():
    n = 40
    row_end, src = chain(n)
    bc = B.scores(row_end, src)
    i = np.arange(n, dtype=np.float64)
    assert np.array_equal(bc, i * (n - 1 - i))


def diamond(double_first=False):
    s, d = [0, 0, 1, 2, 3], [1, 2, 3, 3, 4]
    if double_first:
        s, d = s + [0], d + [1]
    return O.edges_to_csc(5, s, d)


def test_diamond():
    close(B.scores(*diamond()), [0, 1, 1, 3, 0])


def test_diamond_with_a_doubled_edge_counts_multiplicity():
    # from 0: sigma = [1, 2, 1, 3, 3]; delta[3] = 3 * (1/3) = 1, delta[1] = 2 * (1 + 1)/3 = 4/3, delta[2] = 1 * 2/3 = 2/3;
    # sources 1 and 2 each add 1 at vertex 3 (path to 4)
    r = B.run(*diamond(True), [0])
    assert r["sigma"].tolist() == [1, 2, 1, 3, 3]
    close(r["delta"], [r["delta"][0], 4 / 3, 2 / 3, 1, 0])
    close(B.scores(*diamond(True)), [0, 4 / 3, 2 / 3, 3, 0])


def test_two_way_star():
    n = 60
    row_end, src = star(n, both=True)
    bc = B.scores(row_end, src)
    assert bc[0] == (n - 1) * (n - 2) and np.all(bc[1:] == 0)


def test_self_loops_change_nothing():
    row_end, src = rmat(10)
    nv = len(row_end)
    dst = np.repeat(np.arange(nv, dtype=np.int64), np.diff(np.concatenate([[0], row_end]).astype(np.int64)))
    loops = np.arange(0, nv, 3)
    row_end2, src2 = O.edges_to_csc(nv, np.concatenate([src, loops]), np.concatenate([dst, loops]))
    assert np.array_equal(B.scores(row_end, src), B.scores(row_end2, src2))


def test_isolated_source_and_sink_contribute_zero():
    row_end, src = O.edges_to_csc(6, [0, 1, 1], [1, 2, 3])  # 4 and 5 isolated, 2 and 3 sinks
    for s in (4, 2, 3):
        r = B.run(row_end, src, [s])
        assert np.all(r["scores"] == 0) and r["levels"][0] == 1
        assert r["sigma"][s] == 1 and r["sigma"].sum() == 1 and np.all(r["delta"] == 0)
    assert B.scores(row_end, src).tolist() == [0, 2, 0, 0, 0, 0]


@pytest.mark.parametrize("name", ["rmat10", "hand5", "two_components", "trailing_isolated"])
def test_levels_equal_sssp_and_sigma_is_integral(name):
    row_end, src = ALL_SMALL[name]()
    nv = len(row_end)
    for s in (0, nv // 3, nv - 1):
        lev, sigma, delta = B.source_state(row_end, src, s)
        assert np.array_equal(lev, O.label_run(O.APP_SSSP, row_end, src, start=s)["labels"])
        assert np.all(sigma == np.floor(sigma)) and np.all((sigma > 0) == (lev < nv))
        assert np.all(delta[lev == nv] == 0) and np.all(delta >= 0)


def test_multiplicity_counts_on_rmat():
    # RMAT has parallel edges: sigma counts them, so it differs from the de-duplicated graph's somewhere
    row_end, src = rmat(10)
    _, s_multi, _ = B.source_state(row_end, src, 0)
    _, s_dedup, _ = B.source_state(*dedup(row_end, src), 0)
    assert np.any(s_multi != s_dedup) and np.all(s_multi >= s_dedup)


def test_bad_source_is_rejected():
    row_end, src = rmat(8)
    with pytest.raises(ValueError):
        B.run(row_end, src, [len(row_end)])


@pytest.mark.parametrize("make", [B.small_forest, B.forest])
def test_forest_is_exact(make):
    f = make()
    row_end, src, roots = f["row_end"], f["src"], f["roots"]
    nv = len(row_end)
    lev_all = np.full(nv, nv, np.int64)
    for s in roots:
        lev, sigma, delta = B.source_state(row_end, src, s)
        mine = f["tree"] == f["tree"][np.nonzero(np.arange(nv) == s)[0][0]]
        assert np.array_equal(lev[mine], f["level"][mine]) and np.all(lev[~mine] == nv)
        assert np.array_equal(sigma[mine], np.ldexp(1.0, f["log_sigma"][mine]))  # powers of two
        assert np.array_equal(delta[mine], f["descendants"][mine])               # integers
        lev_all[mine] = lev[mine]
    assert np.array_equal(B.scores(row_end, src, roots), f["scores"])
    # every non-root vertex of a tree has exactly one in-neighbour on the previous level; extra edges never go deeper
    dst = np.repeat(np.arange(nv, dtype=np.int64), np.diff(np.concatenate([[0], row_end]).astype(np.int64)))
    lu, lv = lev_all[src.astype(np.int64)], lev_all[dst]
    assert np.all((lu == lv - 1) | (lu >= lv))
    parents = np.unique(np.stack([src[lu == lv - 1].astype(np.int64), dst[lu == lv - 1]], 1), axis=0)
    counts = np.bincount(parents[:, 1], minlength=nv)
    reached = lev_all < nv
    assert np.all(counts[reached & (lev_all > 0)] == 1) and np.all(counts[lev_all == 0] == 0)


def test_forest_has_the_split_cases():
    f = B.forest()
    row_end = f["row_end"]
    indeg = np.diff(np.concatenate([[0], row_end]).astype(np.int64))
    outdeg = np.bincount(f["src"].astype(np.int64), minlength=len(row_end))
    assert outdeg.max() >= 1 << 17          # a hub whose delta sum is cut into segments
    assert indeg.max() >= 1 << 20           # a vertex whose sigma sum is cut into segments (none of them match)
    assert f["level"][f["level"] < len(row_end)].max() >= 2999  # a chain 3000 levels deep
