"""CPU checks of the weighted-SSSP oracle (no GPU).  The reference has no weighted SSSP, so the oracle is pinned by an
independent algorithm: its labels must equal scipy's Dijkstra.  With unit weights it must reproduce the hop-count
oracle (labels and trace), distances saturate at INF = 2^32 - 1, the trace does not depend on the number of partitions,
and the check counts the violations of D[v] <= sat_add(D[u], w)."""
import numpy as np
import pytest
from scipy.sparse import csr_matrix
from scipy.sparse.csgraph import dijkstra

import oracle as O
import weighted_oracle as W
from graphs import ALL_SMALL, rmat

INF = 0xFFFFFFFF


def edge_dst(row_end):
    return np.repeat(np.arange(len(row_end), dtype=np.int64), np.diff(np.concatenate([[0], row_end]).astype(np.int64)))


def scipy_distances(row_end, src, weight, start):
    """Dijkstra from `start` over the edges src[k] -> v with weight[k], as u32 labels with INF = 2^32 - 1.  scipy sums
    duplicate (u, v) entries, so multi-edges are reduced to their minimum weight first; explicit zeros stay edges."""
    nv = len(row_end)
    u = src.astype(np.int64)
    v = edge_dst(row_end)
    w = weight.astype(np.float64)
    if len(u):
        order = np.lexsort((w, v, u))
        u, v, w = u[order], v[order], w[order]
        first = np.ones(len(u), bool)
        first[1:] = (u[1:] != u[:-1]) | (v[1:] != v[:-1])
        u, v, w = u[first], v[first], w[first]  # the smallest weight of every (u, v)
    m = csr_matrix((w, (u, v)), shape=(nv, nv))
    d = dijkstra(m, directed=True, indices=start)
    out = np.full(nv, INF, np.uint64)
    fin = np.isfinite(d)
    out[fin] = np.minimum(d[fin], INF).astype(np.uint64)
    return out.astype(np.uint32)


def random_weights(ne, seed, hi=20):
    return np.random.default_rng(seed).integers(0, hi, ne).astype(np.int32)  # zeros included


def test_hand_graph_equals_dijkstra_and_hand_answer():
    # 0 -> 1 (4), 0 -> 2 (1), 2 -> 1 (2), 1 -> 3 (0), 3 -> 0 (7), 4 -> 3 (1): vertex 4 is unreachable from 0
    row_end, src = O.edges_to_csc(5, [0, 0, 2, 1, 3, 4], [1, 2, 1, 3, 0, 3])
    v = edge_dst(row_end)
    wmap = {(0, 1): 4, (0, 2): 1, (2, 1): 2, (1, 3): 0, (3, 0): 7, (4, 3): 1}
    w = np.array([wmap[(int(s), int(d))] for s, d in zip(src, v)], np.int32)
    ref = W.label_run(row_end, src, w, start=0)
    assert ref["labels"].tolist() == [0, 3, 1, 3, INF]
    assert np.array_equal(ref["labels"], scipy_distances(row_end, src, w, 0))
    assert W.label_check(row_end, src, w, ref["labels"]) == 0


@pytest.mark.parametrize("name", sorted(ALL_SMALL))
def test_small_graphs_random_weights_equal_dijkstra(name):
    row_end, src = ALL_SMALL[name]()
    w = random_weights(len(src), 7)
    for start in (0, len(row_end) - 1):
        ref = W.label_run(row_end, src, w, start=start)
        assert np.array_equal(ref["labels"], scipy_distances(row_end, src, w, start)), (name, start)
        assert W.label_check(row_end, src, w, ref["labels"]) == 0


def test_rmat14_generator_weights_equal_dijkstra():
    seed = 27
    row_end, src = rmat(14, seed=seed)
    w = W.rmat_weights(seed, row_end, src)
    assert w.min() >= 1 and w.max() <= 255
    for start in (0, 77):
        ref = W.label_run(row_end, src, w, start=start)
        assert np.array_equal(ref["labels"], scipy_distances(row_end, src, w, start))
        assert ref["pull"].sum() > 0 and (ref["pull"] == 0).sum() > 0  # both directions taken


@pytest.mark.parametrize("name", sorted(ALL_SMALL))
def test_unit_weights_equal_the_hop_count_oracle(name):
    row_end, src = ALL_SMALL[name]()
    nv = len(row_end)
    ones = np.ones(len(src), np.int32)
    for start in (0, nv - 1):
        hop = O.label_run(O.APP_SSSP, row_end, src, start=start)
        wtd = W.label_run(row_end, src, ones, start=start)
        mapped = np.where(hop["labels"] == nv, np.uint32(INF), hop["labels"])
        assert np.array_equal(wtd["labels"], mapped)
        assert wtd["iters"] == hop["iters"]
        assert np.array_equal(wtd["active"], hop["active"]) and np.array_equal(wtd["pull"], hop["pull"])
        assert np.array_equal(wtd["ftype"], hop["ftype"])


def test_saturation_chain():
    """0 -> 1 -> 2 -> 3 with weights 2^31 - 1, 2^31 - 1, 5: D2 = 2^32 - 2 still fits, D3 would be 2^32 + 3 and is INF
    (no wrap-around to a small distance)."""
    row_end, src = O.edges_to_csc(4, [0, 1, 2], [1, 2, 3])
    w = np.array([2**31 - 1, 2**31 - 1, 5], np.int32)
    ref = W.label_run(row_end, src, w, start=0)
    assert ref["labels"].tolist() == [0, 2**31 - 1, 2**32 - 2, INF]
    assert W.label_check(row_end, src, w, ref["labels"]) == 0
    assert W.sat_add(INF, 0) == INF and W.sat_add(INF, 7) == INF and W.sat_add(INF - 3, 3) == INF
    assert W.sat_add(INF - 3, 2) == INF - 1 and W.sat_add(5, 0) == 5


def test_trace_does_not_depend_on_the_partition_count():
    seed = 5
    row_end, src = rmat(12, seed=seed)
    w = random_weights(len(src), 3, hi=60)
    runs = [W.label_run(row_end, src, w, P=P, start=0) for P in (1, 2, 4)]
    for r in runs[1:]:
        assert np.array_equal(r["labels"], runs[0]["labels"])
        assert r["iters"] == runs[0]["iters"]
        assert np.array_equal(r["active"], runs[0]["active"]) and np.array_equal(r["pull"], runs[0]["pull"])


def test_check_counts_hand_derived_violations():
    # 0 -> 1 (3), 0 -> 2 (1), 2 -> 1 (1), 3 -> 1 (0); vertex 3 unreachable.  Correct: D = [0, 2, 1, INF]
    row_end, src = O.edges_to_csc(4, [0, 0, 2, 3], [1, 2, 1, 1])
    v = edge_dst(row_end)
    wmap = {(0, 1): 3, (0, 2): 1, (2, 1): 1, (3, 1): 0}
    w = np.array([wmap[(int(s), int(d))] for s, d in zip(src, v)], np.int32)
    chk = lambda lab: W.label_check(row_end, src, w, np.array(lab, np.uint32))  # noqa: E731
    assert chk([0, 2, 1, INF]) == 0
    assert chk([0, 5, 1, INF]) == 2      # 0 -> 1 (5 > 3) and 2 -> 1 (5 > 2); 3 -> 1 starts at INF
    assert chk([0, 5, 7, INF]) == 2      # 0 -> 1 and 0 -> 2 (7 > 1); 2 -> 1 holds (5 <= 8)
    assert chk([0, 2, 1, 0]) == 1        # 3 -> 1 now counts: 2 > 0 + 0
    assert chk([INF, INF, INF, INF]) == 0


def rmat_weight_numpy(seed, s, d):
    """Independent restatement of the RMAT weight hash (splitmix64, vectorised)."""
    def splitmix(x):
        z = x + np.uint64(0x9E3779B97F4A7C15)
        z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
        z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
        return z ^ (z >> np.uint64(31))
    with np.errstate(over="ignore"):
        k = splitmix(np.full(1, np.uint64(seed) ^ np.uint64(0x9E3779B97F4A7C15), np.uint64))
        h = splitmix(k ^ ((np.asarray(d, np.uint64) << np.uint64(32)) | np.asarray(s, np.uint64)))
    return (np.uint64(1) + (h >> np.uint64(32)) % np.uint64(255)).astype(np.int32)


def test_rmat_weight_hash_python_equals_c():
    seed = 24
    row_end, src = rmat(12, seed=seed)
    v = edge_dst(row_end)
    w = W.rmat_weights(seed, row_end, src)
    assert np.array_equal(w, rmat_weight_numpy(seed, src, v))
    assert w.min() == 1 and w.max() == 255
    for s, d in ((0, 0), (1, 2), (2, 1), (0xFFFFFFFF, 7)):
        assert W.rmat_weight(seed, s, d) == int(rmat_weight_numpy(seed, [s], [d])[0])
    assert W.rmat_weight(seed, 1, 2) != W.rmat_weight(seed, 2, 1) or W.rmat_weight(seed, 3, 4) != W.rmat_weight(seed, 4, 3)


def test_push_csr_carries_the_weights():
    row_end, src = rmat(10)
    w = random_weights(len(src), 1, hi=1000)
    out_end, out_dst, out_w = W.build_push_csr(row_end, src, w, 0, len(row_end) - 1)
    e2, d2 = O.build_push_csr(row_end, src, 0, len(row_end) - 1)
    assert np.array_equal(out_end, e2) and np.array_equal(out_dst, d2)
    # every (source, destination, weight) triple of the CSC appears once in the CSR
    u_csr = np.repeat(np.arange(len(row_end)), np.diff(np.concatenate([[0], out_end]).astype(np.int64)))
    a = sorted(zip(src.tolist(), edge_dst(row_end).tolist(), w.tolist()))
    b = sorted(zip(u_csr.tolist(), out_dst.tolist(), out_w.tolist()))
    assert a == b
