"""The k-core oracle (tests/kcore_oracle.c) against independent answers, on the CPU: networkx's core_number() on the
undirected simple graph, its two algorithms (Batagelj-Zaversnik and the level-synchronous schedule) against each other,
the closed forms, invariance under how the same graph is stored, the round trace against a numpy restatement of the
schedule, and the check against a numpy restatement of the h-index fixpoint test.  Only the networkx pins need networkx:
without it they skip and the rest still runs."""
import numpy as np
import pytest

import kcore_oracle as K
import tc_oracle as T
from graphs import ALL_SMALL, rmat, symmetrize


def simple_adjacency(row_end, src):
    sp = pytest.importorskip("scipy.sparse")
    nv = len(row_end)
    a, b = T.edges_of(row_end, src)
    keep = a != b
    A = sp.coo_matrix((np.ones(2 * keep.sum(), np.int64), (np.concatenate([a[keep], b[keep]]), np.concatenate([b[keep], a[keep]]))),
                      shape=(nv, nv)).tocsr()
    A.data[:] = 1
    return A


def nx_core(row_end, src):
    nx = pytest.importorskip("networkx")
    a, b = T.edges_of(row_end, src)
    G = nx.Graph()
    G.add_nodes_from(range(len(row_end)))
    G.add_edges_from((int(x), int(y)) for x, y in zip(a, b) if x != y)
    d = nx.core_number(G)
    return np.array([d[v] for v in range(len(row_end))], np.uint32)


def numpy_schedule(row_end, src):
    """The level-synchronous schedule, restated over a scipy CSR with whole-array numpy steps: (core, |F| per round, k
    per round)."""
    A = simple_adjacency(row_end, src)
    nv = A.shape[0]
    deg = np.diff(A.indptr).astype(np.int64)
    alive = np.ones(nv, bool)
    core = np.zeros(nv, np.uint32)
    k, sizes, ks = 0, [], []
    while alive.any():
        k = max(k, int(deg[alive].min()))
        while True:
            f = alive & (deg <= k)
            if not f.any():
                break
            sizes.append(int(f.sum()))
            ks.append(k)
            core[f] = k
            alive &= ~f
            deg -= A @ f.astype(np.int64)
    return core, np.array(sizes, np.uint64), np.array(ks, np.int32)


def numpy_check(row_end, src, core):
    A = simple_adjacency(row_end, src)
    c = core.astype(np.int64)
    rows = np.repeat(np.arange(A.shape[0]), np.diff(A.indptr))
    cu = c[A.indices]
    a = np.bincount(rows, weights=cu >= c[rows], minlength=A.shape[0])
    b = np.bincount(rows, weights=cu >= c[rows] + 1, minlength=A.shape[0])
    return (a < c) | (b >= c + 1)


def check(row_end, src, want=None):
    r = K.run(row_end, src)
    want = nx_core(row_end, src) if want is None else want
    assert np.array_equal(r["core"], want), "core differs at %s" % np.nonzero(r["core"] != want)[0][:10]
    assert np.array_equal(r["core_sync"], want)
    assert r["degeneracy"] == (int(want.max()) if len(want) else 0)
    assert r["rounds"] == len(r["trace_active"]) and int(r["trace_active"].sum()) == len(row_end)
    assert r["levels"] == len(np.unique(r["trace_k"])) and K.check(row_end, src, r["core"])[0] == 0
    return r


@pytest.mark.parametrize("name", sorted(ALL_SMALL))
def test_small_fixtures_vs_networkx(name):
    row_end, src = ALL_SMALL[name]()
    r = check(row_end, src)
    assert r["m"] == simple_adjacency(row_end, src).nnz // 2


@pytest.mark.parametrize("scale", [8, 9, 10, 11, 12])
@pytest.mark.parametrize("form", ["directed", "symmetrised", "duplicated"])
def test_rmat_vs_networkx(scale, form):
    row_end, src = rmat(scale)
    if form == "symmetrised":
        row_end, src = symmetrize(row_end, src)
    elif form == "duplicated":
        row_end, src = T.variant(row_end, src, "mult", seed=scale)
    check(row_end, src)


@pytest.mark.parametrize("scale", [13, 14, 15, 16])
def test_bucket_peel_matches_schedule(scale):
    r = K.run(*rmat(scale))
    assert np.array_equal(r["core"], r["core_sync"]) and r["degeneracy"] == int(r["core"].max())


def test_rmat_schedule_shape():
    """The oracle's RMAT generator at scales 12 and 16: degeneracy, levels, rounds and the widest round."""
    import oracle as O
    for s, want in ((12, (65, 50, 121, 752)), (16, (216, 103, 311, 18685))):
        r = K.run(*O.gen_rmat_csc(s, 1 << s, 16 << s, s))
        assert (r["degeneracy"], r["levels"], r["rounds"], r["max_frontier"]) == want


@pytest.mark.parametrize("name", sorted(K.CLOSED_FORMS))
def test_closed_forms(name):
    row_end, src, core = K.CLOSED_FORMS[name]()
    r = check(row_end, src, core)
    if name == "star":
        assert list(r["trace_active"]) == [1 << 17, 1] and list(r["trace_k"]) == [1, 1]
    if name == "path":
        assert r["rounds"] == 1501 and r["levels"] == 1 and list(r["trace_active"][-2:]) == [2, 1]
    if name == "clique_chain":
        assert r["levels"] == 199 and r["degeneracy"] == 199
    if name == "hub_clique":
        assert list(r["trace_active"]) == [1 << 17, 102] and list(r["trace_k"]) == [1, 101]


def test_small_closed_forms_match_networkx():
    for row_end, src, core in (K.complete(9), K.complete_bipartite(3, 7), K.cycle(11), K.grid(4, 5), K.star(20), K.path(9),
                               K.clique_chain(2, 12), K.hub_clique(7, 30)):
        assert np.array_equal(nx_core(row_end, src), core)


@pytest.mark.parametrize("kind", T.VARIANTS)
def test_noise_invariance(kind):
    for row_end, src in (rmat(11), K.complete(40)[:2], K.clique_chain(2, 30)[:2]):
        base = K.run(row_end, src)
        r = K.run(*T.variant(row_end, src, kind, seed=7))
        assert np.array_equal(r["core"], base["core"]) and r["m"] == base["m"]
        assert np.array_equal(r["trace_active"], base["trace_active"]) and np.array_equal(r["trace_k"], base["trace_k"])


@pytest.mark.parametrize("graph", ["rmat10", "rmat13_sym", "clique_chain", "star"])
def test_trace_vs_numpy_schedule(graph):
    if graph == "clique_chain":
        row_end, src = K.clique_chain(2, 40)[:2]
    elif graph == "star":
        row_end, src = K.star(500)[:2]
    elif graph.endswith("_sym"):
        row_end, src = symmetrize(*rmat(13))
    else:
        row_end, src = rmat(10)
    r = K.run(row_end, src)
    core, sizes, ks = numpy_schedule(row_end, src)
    assert np.array_equal(r["core_sync"], core)
    assert np.array_equal(r["trace_active"], sizes) and np.array_equal(r["trace_k"], ks)


def test_check_on_planted_corruptions():
    row_end, src = rmat(12)
    good = K.run(row_end, src)["core"]
    rng = np.random.default_rng(5)
    cases = []
    for _ in range(6):  # +-1 at one vertex of degree > 0
        bad = good.copy()
        v = int(rng.choice(np.nonzero(good > 0)[0]))
        bad[v] = int(good[v]) + (1 if rng.random() < 0.5 else -1)  # v itself always violates
        cases.append(bad)
    cases.append(rng.permutation(good))
    for core in cases:
        n, mask = K.check(row_end, src, core)
        want = numpy_check(row_end, src, core)
        assert n > 0 and np.array_equal(mask, want)
    # all zeros pass: the check is necessary, not sufficient (core numbers are the largest fixpoint)
    zeros = np.zeros_like(good)
    assert K.check(row_end, src, zeros)[0] == 0 and not numpy_check(row_end, src, zeros).any()
    assert K.check(row_end, src, good)[0] == 0 and not numpy_check(row_end, src, good).any()


def test_edgeless_and_bad_source():
    row_end = np.zeros(5, np.uint64)
    r = K.run(row_end, np.zeros(0, np.uint32))
    assert r["degeneracy"] == 0 and r["rounds"] == 1 and not r["core"].any()
    r = K.run(np.array([1, 2], np.uint64), np.array([0, 1], np.uint32))  # self-loops only
    assert r["degeneracy"] == 0 and list(r["trace_active"]) == [2]
    with pytest.raises(ValueError):
        K.run(np.array([1, 1], np.uint64), np.array([5], np.uint32))
