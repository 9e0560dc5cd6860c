"""The k-truss oracle (tests/truss_oracle.c) against independent answers, on the CPU: networkx's k_truss(G, k) for every
k, the support against scipy's (A @ A) ∘ A, its two peels (Wang-Cheng buckets and the level-synchronous schedule) against
each other, the closed forms, invariance under how the same graph is stored, and the check against a numpy restatement.
Only the networkx pins need networkx: without it they skip and the rest still runs."""
import numpy as np
import pytest

import tc_oracle as T
import truss_oracle as R
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


def nx_truss(row_end, src, lo, hi):
    """τ per edge from networkx: the largest k whose k_truss holds the edge."""
    nx = pytest.importorskip("networkx")
    a, b = T.edges_of(row_end, src)
    G = nx.Graph()
    G.add_nodes_from(range(len(row_end)))
    G.add_edges_from((int(x), int(y)) for x, y in zip(a, b) if x != y)
    tau = np.zeros(len(lo), np.uint32)
    index = {(int(x), int(y)): i for i, (x, y) in enumerate(zip(lo, hi))}
    k = 2
    H = G
    while H.number_of_edges():
        H = nx.k_truss(H, k)
        for x, y in H.edges():
            tau[index[(min(x, y), max(x, y))]] = k
        k += 1
    return tau


def numpy_check(row_end, src, lo, hi, tau):
    A = simple_adjacency(row_end, src)
    nv = A.shape[0]
    T_ = A.tolil()
    for i, (x, y) in enumerate(zip(lo, hi)):
        T_[x, y] = T_[y, x] = int(tau[i]) + 1  # stored +1: zero is absent in a sparse matrix
    T_ = T_.tocsr()
    bad = np.zeros(len(lo), bool)
    for i, (x, y) in enumerate(zip(lo, hi)):
        c = int(tau[i])
        rx, ry = T_.getrow(x), T_.getrow(y)
        common = np.intersect1d(rx.indices, ry.indices)
        t = np.minimum(rx[0, common].toarray().ravel(), ry[0, common].toarray().ravel()) - 1 if len(common) else np.zeros(0)
        a, b = int((t >= c).sum()), int((t >= c + 1).sum())
        bad[i] = c < 2 or a < c - 2 or b >= c - 1
    assert nv == len(row_end)
    return bad


def check(row_end, src, want=None):
    r = R.run(row_end, src)
    want = nx_truss(row_end, src, r["lo"], r["hi"]) if want is None else want
    assert np.array_equal(r["truss"], want), "truss differs at %s" % np.nonzero(r["truss"] != want)[0][:10]
    assert np.array_equal(r["truss_sync"], want)
    assert r["kmax"] == (int(want.max()) if len(want) else 0)
    assert r["rounds"] == len(r["trace_active"]) and int(r["trace_active"].sum()) == r["m"]
    assert r["levels"] == len(np.unique(r["trace_k"])) and R.check(row_end, src, r["truss"])[0] == 0
    assert np.all(r["lo"] < r["hi"]) and np.all(np.diff(r["lo"].astype(np.int64) << 32 | r["hi"]) > 0)
    tv = np.zeros(len(row_end), np.uint32)
    np.maximum.at(tv, r["lo"], r["truss"])
    np.maximum.at(tv, r["hi"], r["truss"])
    assert np.array_equal(r["vertex"], tv)
    return r


@pytest.mark.parametrize("name", sorted(ALL_SMALL))
def test_small_fixtures_vs_networkx(name):
    check(*ALL_SMALL[name]())


@pytest.mark.parametrize("scale", [8, 9, 10])  # networkx's k_truss takes about 90 s per graph at RMAT-12
@pytest.mark.parametrize("form", ["directed", "symmetrised", "duplicated"])
def test_rmat_vs_networkx(scale, form):
    row_end, src = rmat(scale)
    if form == "symmetrised":
        row_end, src = symmetrize(row_end, src)
    elif form == "duplicated":
        row_end, src = T.variant(row_end, src, "mult", seed=scale)
    check(row_end, src)


@pytest.mark.parametrize("scale", [10, 12, 14, 16])
def test_support_vs_scipy(scale):
    row_end, src = rmat(scale)
    r = R.run(row_end, src)
    A = simple_adjacency(row_end, src)
    S = (A @ A).multiply(A).tocsr()
    assert r["m"] == A.nnz // 2
    want = np.asarray(S[r["lo"], r["hi"]]).ravel()
    assert np.array_equal(r["support"], want)


@pytest.mark.parametrize("scale", [13, 14, 15, 16])
def test_bucket_peel_matches_schedule(scale):
    r = R.run(*rmat(scale))
    assert np.array_equal(r["truss"], r["truss_sync"]) and r["kmax"] == int(r["truss"].max())


@pytest.mark.parametrize("name", sorted(R.CLOSED_FORMS))
def test_closed_forms(name):
    row_end, src, tau = R.CLOSED_FORMS[name]()
    r = check(row_end, src, tau)
    if name == "k48":
        assert r["rounds"] == 1 and np.all(r["support"] == 46)
    if name == "book":
        assert list(r["trace_active"]) == [1 << 18, 1] and r["support"][0] == 1 << 17
    if name == "wheel":
        assert list(r["trace_active"]) == [1000, 1000] and list(r["trace_k"]) == [3, 3]
    if name in ("k_30_45", "cycle", "grid"):
        assert r["rounds"] == 1 and r["kmax"] == 2
    if name == "tube":
        assert r["rounds"] == 3000 and set(r["trace_k"]) == {3}
    if name == "cliques":
        assert r["levels"] == 28 and r["kmax"] == 30
    if name == "no_edges":
        assert r["m"] == 0 and r["rounds"] == 0 and r["kmax"] == 0 and not r["vertex"].any()


def test_clique_result_in_closed_form():
    """The closed-form K_n result the GPU test uses for K_2048, against the oracle at a size it runs quickly."""
    row_end, src, _ = R.complete(40)
    r, want = R.run(row_end, src), R.clique_result(40)
    for key, value in want.items():
        assert np.array_equal(np.asarray(r[key]), np.asarray(value)), key


def test_small_closed_forms_match_networkx():
    for row_end, src, tau in (R.complete(9), R.cliques(8), R.book(20), R.wheel(12), R.complete_bipartite(3, 7), R.cycle(11),
                              R.grid(4, 5), R.tube(100), R.tube(300)):
        r = R.run(row_end, src)
        assert np.array_equal(nx_truss(row_end, src, r["lo"], r["hi"]), tau)


@pytest.mark.parametrize("kind", T.VARIANTS)
def test_noise_invariance(kind):
    for row_end, src in (rmat(11), R.complete(40)[:2], R.cliques(12)[:2]):
        base = R.run(row_end, src)
        r = R.run(*T.variant(row_end, src, kind, seed=7))
        for key in ("lo", "hi", "support", "truss", "trace_active", "trace_k"):
            assert np.array_equal(r[key], base[key]), key


def test_check_on_planted_corruptions():
    row_end, src = rmat(10)
    r = R.run(row_end, src)
    good, lo, hi = r["truss"], r["lo"], r["hi"]
    rng = np.random.default_rng(5)
    cases = []
    for _ in range(6):  # +-1 on one edge
        bad = good.copy()
        e = int(rng.integers(len(good)))
        bad[e] = int(good[e]) + (1 if rng.random() < 0.5 else -1)
        cases.append(bad)
    cases += [rng.permutation(good), np.full_like(good, 0xFFFFFFFF)]
    for tau in cases:
        n, mask = R.check(row_end, src, tau)
        assert n > 0 and np.array_equal(mask, numpy_check(row_end, src, lo, hi, tau))
    # all 2s pass: the check is necessary, not sufficient
    twos = np.full_like(good, 2)
    assert R.check(row_end, src, twos)[0] == 0 and not numpy_check(row_end, src, lo, hi, twos).any()
    assert R.check(row_end, src, good)[0] == 0


def test_bad_source():
    with pytest.raises(ValueError):
        R.run(np.array([1, 1], np.uint64), np.array([5], np.uint32))
