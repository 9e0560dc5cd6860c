"""Small deterministic input graphs shared by the oracle tests and the GPU parity tests (built with the oracle)."""
import numpy as np

import oracle as O


def hand5():
    """The 5-edge graph whose .lux bytes SURVEY §8f-1 verified against tools/converter.cc:
    edges {0->1, 1->2, 2->0, 3->0, 0->2}."""
    return O.edges_to_csc(4, [0, 1, 2, 3, 0], [1, 2, 0, 0, 2])


def star(n=10000, both=True):
    """Hub: every vertex -> 0 (in-degree n-1 spans several merge tiles); optionally 0 -> every vertex."""
    s = list(range(1, n))
    d = [0] * (n - 1)
    if both:
        s += [0] * (n - 1)
        d += list(range(1, n))
    return O.edges_to_csc(n, s, d)


def chain(n=3000, symmetric=False):
    s = list(range(0, n - 1))
    d = list(range(1, n))
    if symmetric:
        s, d = s + d, d + s
    return O.edges_to_csc(n, s, d)


def no_edges(n=7):
    return np.zeros(n, np.uint64), np.zeros(0, np.uint32)


def trailing_isolated(n_core=500, n_iso=5000, seed=9):
    """RMAT core followed by a long tail of vertices with no edges at all (ragged tiles: all-vertex tiles)."""
    re, src = O.gen_rmat_csc(9, n_core, 8 * n_core, seed)
    re2 = np.concatenate([re, np.full(n_iso, re[-1], np.uint64)])
    return re2, src


def rmat(scale, ef=16, seed=27, nv=None):
    nv = (1 << scale) if nv is None else nv
    return O.gen_rmat_csc(scale, nv, ef * nv, seed)


def symmetrize(row_end, src):
    nv = len(row_end)
    dst = np.repeat(np.arange(nv, dtype=np.uint32), np.diff(np.concatenate([[0], row_end]).astype(np.int64)))
    return O.edges_to_csc(nv, np.concatenate([src, dst]), np.concatenate([dst, src]))


def two_components(n=2000):
    """Two disjoint symmetric chains + isolated vertices: CC must label them max-id per component."""
    h = n // 2
    s = list(range(0, h - 1)) + list(range(h, n - 11))
    d = list(range(1, h)) + list(range(h + 1, n - 10))
    return O.edges_to_csc(n, s + d, d + s)


def in_degrees(row_end):
    return np.diff(np.concatenate([[0], row_end]).astype(np.int64))


def mix32(ids, salt=0):
    """A fixed 32-bit hash of vertex ids (splitmix64 finaliser, vectorised): spreads test values over the sources."""
    z = np.asarray(ids).astype(np.uint64) + np.uint64(((salt + 1) * 0x9E3779B97F4A7C15) & (2**64 - 1))
    z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
    z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
    return (z ^ (z >> np.uint64(31))) >> np.uint64(32)


def exact_pr_inputs(nv, max_indeg, passes=4, salt=0):
    """PageRank values on which every summation order is exact: integers cast to float32, so that one iteration from
    them must equal the oracle's bit for bit whatever the sweep's reduction shape.

    The largest raw sum S = sum of x[u] over a vertex's in-edges stays below 2^21: fp32 lane sums, shuffle scans and
    partials of integers are then exact, and S off by one moves fma(0.15, S, init) by more than two ulps, which
    survives the division by the out-degree.  Values x in {1..K}, K = floor(2^20 / max_indeg), make every edge count
    and most misrouted sources visible in one pass.  Where K = 1 (a hub with more than 2^19 in-edges), `passes`
    inputs: all ones (counts edges), then single hash bits of u in {0, 1} (finds misrouted sources).  `salt` picks
    another set of values of the same kind."""
    assert max_indeg < (1 << 21), "in-degree %d: sums of ones are no longer exact enough" % max_indeg
    h = mix32(np.arange(nv, dtype=np.uint64), salt)
    k = (1 << 20) // max(int(max_indeg), 1)
    if k >= 2:
        return [(np.uint64(1) + h % np.uint64(k)).astype(np.float32)]
    return [np.ones(nv, np.float32)] + [((h >> np.uint64(b)) & np.uint64(1)).astype(np.float32) for b in range(passes - 1)]


def exact_cf_inputs(users, items, max_item_indeg):
    """Collaborative-filtering vectors on which every dot product, error, err * x_u and chunk sum is exact: users get
    integers in {1, 2} on all 20 factors, items integers in {1..b} on factors 0-9 and zeros on factors 10-19.  Every
    user -> item edge then has dot >= 10 > rating, so err < 0 and all terms of an item's accumulator have one sign:
    its partial sums never exceed the final |acc|, which b keeps below 2^22 (|err * x_u| <= 2 * 20 b per edge).
    For an item, factors 10-19 come out as rn(GAMMA * acc): bit-exact whether or not the update is contracted to an
    FMA, and a function of the weight, the dot product and the source of every in-edge."""
    b = int(min(8, max(1, (1 << 22) // (40 * max(int(max_item_indeg), 1)))))
    x = np.zeros((users + items, 20), np.float32)
    uid = np.arange(users, dtype=np.uint64)
    x[:users] = (np.uint64(1) + ((mix32(uid, 1)[:, None] >> np.arange(20, dtype=np.uint64)) & np.uint64(1))).astype(np.float32)
    iid = np.arange(items, dtype=np.uint64)
    x[users:, :10] = (np.uint64(1) + (mix32(iid, 2)[:, None] >> (np.uint64(3) * np.arange(10, dtype=np.uint64))) % np.uint64(b)).astype(np.float32)
    return x


ALL_SMALL = {
    "hand5": hand5,
    "star": star,
    "chain": chain,
    "no_edges": no_edges,
    "trailing_isolated": trailing_isolated,
    "rmat10": lambda: rmat(10),
    "rmat12_ragged_nv": lambda: rmat(12, nv=3000),
    "two_components": two_components,
}
