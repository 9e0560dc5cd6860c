"""The triangle-counting oracle (tests/tc_oracle.c) against independent answers, on the CPU: networkx's triangles() on the
undirected simple graph, scipy's ((A @ A) .* A) row sums on the simple adjacency, the closed forms of the exact inputs
(K_n, wheels, windmills, K_{p,q}, the over-budget graph), and invariance under how the same graph is stored."""
import numpy as np
import pytest

import tc_oracle as T
from graphs import ALL_SMALL, rmat, symmetrize

nx = pytest.importorskip("networkx")
sp = pytest.importorskip("scipy.sparse")


def nx_triangles(row_end, src):
    a, b = T.edges_of(row_end, src)
    G = nx.Graph()
    G.add_nodes_from(range(len(row_end)))
    G.add_edges_from((int(x), int(y)) for x, y in zip(a, b) if x != y)
    d = nx.triangles(G)
    return np.array([d[v] for v in range(len(row_end))], np.uint64)


def simple_adjacency(row_end, src):
    nv = len(row_end)
    a, b = T.edges_of(row_end, src)
    keep = a != b
    A = sp.coo_matrix((np.ones(2 * keep.sum(), np.int64), (np.concatenate([a[keep], b[keep]]), np.concatenate([b[keep], a[keep]]))),
                      shape=(nv, nv)).tocsr()
    A.data[:] = 1  # duplicates summed by the conversion collapse to one edge
    return A


def scipy_triangles(row_end, src):
    A = simple_adjacency(row_end, src)
    return (np.asarray((A @ A).multiply(A).sum(axis=1)).ravel() // 2).astype(np.uint64), A.nnz // 2


def check(row_end, src, want):
    r = T.run(row_end, src)
    assert np.array_equal(r["t"], want), "t differs at %s" % np.nonzero(r["t"] != want)[0][:10]
    assert 3 * r["total"] == int(want.sum())
    return r


@pytest.mark.parametrize("name", sorted(ALL_SMALL))
def test_small_fixtures_vs_networkx(name):
    row_end, src = ALL_SMALL[name]()
    r = check(row_end, src, nx_triangles(row_end, src))
    assert r["m"] == simple_adjacency(row_end, src).nnz // 2


@pytest.mark.parametrize("scale", [8, 9, 10, 11, 12])
@pytest.mark.parametrize("form", ["directed", "symmetrised", "duplicated"])
def test_rmat_vs_networkx(scale, form):
    row_end, src = rmat(scale)
    if form == "symmetrised":
        row_end, src = symmetrize(row_end, src)
    elif form == "duplicated":
        row_end, src = T.variant(row_end, src, "mult", seed=scale)
    check(row_end, src, nx_triangles(row_end, src))


@pytest.mark.parametrize("scale", [14, 15, 16])
def test_rmat_vs_scipy(scale):
    row_end, src = rmat(scale)
    want, m = scipy_triangles(row_end, src)
    r = check(row_end, src, want)
    assert r["m"] == m and r["total"] > 0


def test_closed_forms():
    for n in (1, 2, 3, 4, 10, 60):
        check(*T.complete(n))
    for rim in (4, 5, 100, 1000):
        check(*T.wheel(rim))
    for k in (1, 2, 50, 3000):
        check(*T.windmill(k))
    for p, q in ((1, 1), (3, 5), (40, 70)):
        check(*T.complete_bipartite(p, q))
    for B, H in ((16, 3), (64, 34), (100, 1)):
        row_end, src, t = T.over_budget(B, H)
        r = check(row_end, src, t)
        assert r["total"] == H * (B + 9) and r["max_out"] == B + 4


def test_closed_forms_match_networkx():
    for row_end, src, t in (T.complete(12), T.wheel(17), T.windmill(9), T.complete_bipartite(6, 7), T.over_budget(16, 5)):
        assert np.array_equal(nx_triangles(row_end, src), t)


@pytest.mark.parametrize("kind", T.VARIANTS)
def test_noise_invariance(kind):
    for row_end, src in (rmat(11), T.complete(40)[:2], T.wheel(300)[:2]):
        base = T.run(row_end, src)
        r = T.run(*T.variant(row_end, src, kind, seed=7))
        assert np.array_equal(r["t"], base["t"]) and r["total"] == base["total"] and r["m"] == base["m"]
        assert r["probes"] == base["probes"]


def test_probe_count_and_orientation():
    # K_n under degree order = id order: |N+(u)| = n - 1 - u, probes = sum over u < v of (n - 1 - v)
    n = 30
    r = T.run(*T.complete(n)[:2])
    assert r["max_out"] == n - 1
    assert r["probes"] == sum(n - 1 - v for u in range(n) for v in range(u + 1, n))
    # degree order bounds every out-list by sqrt(2m)
    r = T.run(*rmat(14))
    assert r["max_out"] <= int(np.sqrt(2 * r["m"])) + 1


def test_bad_source_id():
    row_end = np.array([1, 1], np.uint64)
    with pytest.raises(ValueError):
        T.run(row_end, np.array([5], np.uint32))
