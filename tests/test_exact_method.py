"""The exact-input method of tests/test_gpu_exact.py, proved on the CPU with the oracle alone.

The GPU parity tests compare PageRank at 1e-6 relative and CF at 2e-6: on ordinary inputs an fp32 sweep cannot match
the oracle's fp64 sum bit for bit.  Those tolerances are wider than one wrong edge into a large hub.  On the integer
inputs of graphs.exact_pr_inputs / exact_cf_inputs every summation order is exact, so the comparison can be
np.array_equal — and these tests show that it then sees a dropped, a duplicated and a re-pointed edge, all made in the
oracle's own CSC, where the tolerance comparison on ordinary values does not."""
import numpy as np

import oracle as O
from graphs import exact_cf_inputs, exact_pr_inputs, in_degrees

CF_GAMMA = np.float32(0.00000035)


def star_csc(n_in):
    """Vertex 0 has n_in in-edges, from vertices 1 .. n_in; no other edges."""
    row_end = np.full(n_in + 1, n_in, np.uint64)
    src = np.arange(1, n_in + 1, dtype=np.uint32)
    return row_end, src


def dropped(row_end, src, k):
    re2 = row_end.copy()
    re2[np.searchsorted(row_end, k, side="right"):] -= 1
    return re2, np.delete(src, k)


def duplicated(row_end, src, k):
    re2 = row_end.copy()
    re2[np.searchsorted(row_end, k, side="right"):] += 1
    return re2, np.insert(src, k, src[k])


def repointed(src, k, new_src):
    s2 = src.copy()
    s2[k] = new_src
    return s2


def within(a, b, rtol):
    a64, b64 = a.astype(np.float64), b.astype(np.float64)
    return bool(np.all(np.abs(a64 - b64) <= rtol * np.abs(b64)))


def test_exact_pagerank_inputs_see_one_wrong_edge_into_a_2m_hub():
    n_in = 2_000_000
    row_end, src = star_csc(n_in)
    nv = len(row_end)
    deg = O.out_degree(nv, src)  # the kernel's degrees stay those of the true graph
    xs = exact_pr_inputs(nv, int(in_degrees(row_end).max()))
    assert len(xs) > 1 and np.array_equal(xs[0], np.ones(nv, np.float32))  # K = 1: counting pass + source-bit passes
    want = [O.pagerank_iter(row_end, src, deg, x) for x in xs]
    k = 1_234_567

    def caught(re2, src2):
        return any(not np.array_equal(O.pagerank_iter(re2, src2, deg, x), w) for x, w in zip(xs, want))

    assert caught(*dropped(row_end, src, k))
    assert caught(*duplicated(row_end, src, k))
    assert caught(row_end, repointed(src, k, src[k] + 1))
    assert not caught(row_end, src)
    # the same drop on ordinary PageRank values passes a 1e-6 comparison
    x0 = O.pagerank_init(deg)
    ok = O.pagerank_iter(row_end, src, deg, x0)
    assert within(O.pagerank_iter(*dropped(row_end, src, k), deg, x0), ok, 1e-6)


def test_exact_cf_inputs_see_a_repointed_source():
    users, items = 300, 40
    row_end, src, w = O.gen_bipartite_csc(users, items, 20000, 5)
    indeg = in_degrees(row_end)
    item0 = users + int(np.argmax(indeg[users:]))  # the largest item
    e0 = int(row_end[item0 - 1]) if item0 else 0
    k = e0 + int(indeg[item0]) // 2
    other = (int(src[k]) + 1) % users
    src2 = repointed(src, k, other)
    # ordinary values: at 1 and 3 iterations a wrong source index is invisible at 2e-6
    for ni in (1, 3):
        assert within(O.colfilter(row_end, src2, w, ni), O.colfilter(row_end, src, w, ni), 2e-6)
    # exact inputs: the item's factors 10-19 are rn(GAMMA * acc) with |acc| < 2^22, and they move
    x = exact_cf_inputs(users, items, int(indeg[users:].max()))
    ok = O.cf_iter(row_end, src, w, x)
    assert np.abs(ok[users:, 10:]).max() / CF_GAMMA < (1 << 22) * (1 - 1e-6)
    bad = O.cf_iter(row_end, src2, w, x)
    assert not np.array_equal(bad[item0, 10:], ok[item0, 10:])
    assert np.array_equal(bad[users:, 10:][np.arange(items) != item0 - users], ok[users:, 10:][np.arange(items) != item0 - users])
