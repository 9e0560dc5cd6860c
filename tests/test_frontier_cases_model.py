"""Designed graphs for the CC / SSSP frontier engine (push.cuh, label_iteration in api.cu), each aimed at one boundary of
the push and queue logic, and the CPU checks that every case hits the boundary it is named after.  A rule that drifts
then fails here as a configuration error instead of letting tests/test_gpu_frontier.py pass without reaching the code.

The GPU test compares the device after EVERY iteration with the Jacobi sequence L_{k+1} = label_pull(L_k): the push
reads the iteration-start labels and relaxes a working copy, so the labels after an iteration do not depend on the
direction, and a vertex inactive in iteration k already contributed its label to L_k.  This file checks that claim on
the oracle (`label_run`'s labels, iteration count and active counts against iterated `label_pull`), together with the
direction and representation rules on one rank: iteration k pulls iff the frontier it starts from has more than nv/16
vertices; its new frontier is a bitmap iff it has at least cap = (nv - 1)/16 + 100 vertices (promotion after a push,
demotion after a pull: on one rank both reduce to that count)."""
import numpy as np
import pytest

import oracle as O
import weighted_oracle as W
from graphs import ALL_SMALL, rmat, symmetrize

CC, SSSP, WSSSP = "cc", "sssp", "wsssp"
APPS = (CC, SSSP, WSSSP)
NV = 1 << 16


def cap(nv):
    """Frontier queue capacity of a one-rank partition, (R - L)/16 + 100 (push_model.inl:393)."""
    return (nv - 1) // 16 + 100


def case_weights(src, seed=1):
    """Weights in CSC order for the weighted runs: small integers, zeros included (ties and zero-cost hops)."""
    return np.random.default_rng(seed).integers(0, 8, len(src)).astype(np.int32)


class Graph:
    def __init__(self, nv, esrc, edst, marks=None, seed=1):
        self.row_end, self.src = O.edges_to_csc(nv, esrc, edst)
        self.weight = case_weights(self.src, seed)
        self.marks = marks or {}  # vertex sets the boundary asserts refer to
        self.nv = nv


def _arr(*parts):
    return np.concatenate([np.asarray(p, np.int64).ravel() for p in parts])


# ---- the cases -----------------------------------------------------------------------------------------------------

BIG_DEGREES = (2047, 2048, 2049, 4096, 4097, 8192, 8193, 3 * 4096 + 1)
POOL_LO, POOL_N = 100, 4000


def big_source_degrees():
    """H = nv-1 -> m -> B (8 sources of the degrees above) -> a shared pool of 4000 destinations, each source also
    reaching one private destination with its LAST out-edge (the tail segment of a hub).  The 8193-edge source carries
    a self-loop and duplicate edges (its pool edges wrap around).  CC: only m changes in the first (pull) iteration,
    B in the second, the pool in the third; SSSP from H the same: B relaxes the pool in a push iteration, the inline
    kernel (2047, 2048) and the segment kernel on the same destinations."""
    nv = NV
    H, m = nv - 1, 10
    B = 20 + np.arange(len(BIG_DEGREES))
    s, d = [[H], [m] * len(B)], [[m], B]
    for i, (b, deg) in enumerate(zip(B, BIG_DEGREES)):
        own = [b] if deg == 8193 else []  # self-loop
        n_pool = deg - 1 - len(own)
        pool = POOL_LO + (i * 517 + np.arange(n_pool)) % POOL_N
        s.append(np.full(deg, b))
        d.append(_arr(own, pool, [nv - 2 - i]))
    return Graph(nv, _arr(*s), _arr(*d), dict(big=B))


def fan(T, per_source=None, second=False):
    """H = nv-1 -> sources -> T destinations 1000.. : the second iteration (a push, from the sources) changes exactly
    T vertices.  One source of out-degree T (the segment kernel), or sources of per_source out-edges plus 3 of the
    previous source's (overlapping, all inline).  second: destination j -> 20000 + j, so the iteration after that has
    T sources of its own."""
    nv = NV
    H = nv - 1
    dst = 1000 + np.arange(T)
    if per_source is None:
        srcs = np.array([5])
        s, d = [np.full(T, 5)], [dst]
    else:
        k = -(-T // per_source)
        srcs = 1 + np.arange(k)
        s, d = [], []
        for j in range(k):
            lo = max(j * per_source - 3, 0)
            hi = min((j + 1) * per_source, T)
            s.append(np.full(hi - lo, srcs[j]))
            d.append(dst[lo:hi])
    s, d = [np.full(len(srcs), H)] + s, [srcs] + d
    if second:
        s.append(dst)
        d.append(20000 + np.arange(T))
    return Graph(nv, _arr(*s), _arr(*d), dict(sources=srcs, dests=dst))


def demotion(c):
    """CC: nv-1 -> c targets, so the first (pull) iteration changes exactly c vertices.  SSSP from 0: 0 -> A (4200
    vertices, a push that promotes), then a pull iteration A[j] -> target j that changes exactly c.  The targets are
    shared by both paths (A's ids are below nv-1, so in CC they change nothing)."""
    nv = NV
    A = 1000 + np.arange(4200)
    T = 10000 + np.arange(c)
    return Graph(nv, _arr(np.full(c, nv - 1), np.zeros(len(A)), A[:c]), _arr(T, A, T), dict(targets=T))


def contention(K, M):
    """0 -> H_i -> s_i -> every d_j (complete bipartite K x M).  CC: s_i takes H_i = nv - K + i in the first (pull)
    iteration, then K distinct candidates race for each d_j in a push.  SSSP from 0: equal candidates (hop 3)."""
    nv = NV
    Hs = nv - K + np.arange(K)
    S = 1000 + np.arange(K)
    D = 2000 + np.arange(M)
    return Graph(nv, _arr(np.zeros(K), Hs, np.repeat(S, M)), _arr(Hs, S, np.tile(D, K)), dict(sources=S, dests=D))


def ragged():
    """nv = 5003 (not a multiple of 8 or 32: the last bitmap word and byte are partial), symmetrised RMAT."""
    return Graph(5003, *_edges(symmetrize(*rmat(13, ef=4, nv=5003))))


def tiny():
    """nv = 13 < 16: nv/16 = 0, every iteration pulls.  A chain with back edges; 12 has no out-edges."""
    s = list(range(12)) + [3, 7, 11]
    d = list(range(1, 13)) + [1, 2, 5]
    return Graph(13, s, d)


def sink_start():
    """nv = 1000 (nv/16 = 62, a frontier of one pushes): 999 has in-edges and no out-edges."""
    rng = np.random.default_rng(5)
    s = rng.integers(0, 999, 6000)
    d = rng.integers(0, 1000, 6000)
    return Graph(1000, s, d)


def _edges(csc):
    row_end, src = csc
    dst = np.repeat(np.arange(len(row_end)), np.diff(np.concatenate([[0], row_end]).astype(np.int64)))
    return src, dst


C = cap(NV)
# name -> (builder, runs ((app, start), ...), boundary assert (graph, app, ref) -> None)
CASES = {}


def _case(name, builder, runs, expect):
    CASES[name] = (builder, tuple(runs), expect)


def _all(start):
    return [(CC, 0), (SSSP, start), (WSSSP, start)]


def changed(ref, k):
    """Vertices whose label iteration k changed."""
    return np.nonzero(ref.labels[k + 1] != ref.labels[k])[0]


def expect_big(g, app, ref):
    deg = O.out_degree(g.nv, g.src)
    assert deg[g.marks["big"]].tolist() == list(BIG_DEGREES)
    hits = [k for k in range(1, ref.iters) if not ref.pull[k] and np.array_equal(changed(ref, k - 1), np.sort(g.marks["big"]))]
    assert hits and ref.active[hits[0]] == POOL_N + len(BIG_DEGREES), "no push iteration from exactly the big sources"


_case("big_source_degrees", big_source_degrees, _all(NV - 1), expect_big)


def expect_fan(T, one_source):
    def check(g, app, ref):
        k = [k for k in range(1, ref.iters) if np.array_equal(changed(ref, k - 1), g.marks["sources"])]
        assert k, "the sources never form a frontier"
        k = k[0]
        assert not ref.pull[k] and ref.active[k] == T
        assert ref.ftype[k] == (O.SPARSE_QUEUE if T < C else O.DENSE_BITMAP)
        deg = O.out_degree(g.nv, g.src)[g.marks["sources"]]
        assert (deg == T).all() if one_source else (len(deg) > 1 and deg.max() <= 2048)
    return check


for _T in (C - 1, C, C + 1, C + 31, C + 33):
    _case("queue_at_capacity_one_hub_%+d" % (_T - C), lambda T=_T: fan(T), _all(NV - 1), expect_fan(_T, True))
    _case("queue_at_capacity_many_%+d" % (_T - C), lambda T=_T: fan(T, per_source=40), _all(NV - 1), expect_fan(_T, False))


def expect_direction(T):
    def check(g, app, ref):
        k = [k for k in range(ref.iters) if np.array_equal(changed(ref, k), g.marks["dests"])]
        assert k and k[0] + 1 < ref.iters, "the destinations never form a frontier"
        k = k[0]
        assert ref.active[k] == T and ref.active[k + 1] == T
        assert ref.pull[k + 1] == (T > NV // 16)
    return check


for _T in (NV // 16, NV // 16 + 1):
    _case("direction_threshold_%d" % _T, lambda T=_T: fan(T, per_source=40, second=True), _all(NV - 1), expect_direction(_T))


def expect_demotion(c):
    def check(g, app, ref):
        k = [k for k in range(ref.iters) if np.array_equal(changed(ref, k), g.marks["targets"])]
        assert k, "the targets never change together"
        k = k[0]
        assert ref.pull[k] and ref.active[k] == c
        assert ref.ftype[k] == (O.SPARSE_QUEUE if c < C else O.DENSE_BITMAP)
        if app != CC:
            assert ref.ftype[k - 1] == O.DENSE_BITMAP and not ref.pull[k - 1]  # the push before it promoted
    return check


for _c in (C - 1, C):
    _case("demotion_at_capacity_%+d" % (_c - C), lambda c=_c: demotion(c), _all(0), expect_demotion(_c))


def expect_contention(K, M):
    def check(g, app, ref):
        S, D = g.marks["sources"], g.marks["dests"]
        k = [k for k in range(1, ref.iters) if np.array_equal(changed(ref, k - 1), S)]
        assert k, "the sources never form a frontier"
        k = k[0]
        assert not ref.pull[k] and ref.active[k] == M and np.array_equal(changed(ref, k), D)
        cand = ref.labels[k][S]
        if app == CC:
            assert len(np.unique(cand)) == K
        elif app == SSSP:
            assert len(np.unique(cand)) == 1
    return check


for _K, _M in ((64, 1500), (64, 3000)):
    _case("exactly_once_contention_%dx%d" % (_K, _M), lambda K=_K, M=_M: contention(K, M), _all(0), expect_contention(_K, _M))


def expect_ragged(g, app, ref):
    assert g.nv % 8 and g.nv % 32
    tail = g.nv - g.nv % 32
    assert any(ref.ftype[k] == O.DENSE_BITMAP and (changed(ref, k) >= tail).any() for k in range(ref.iters))


_case("ragged_nv", ragged, [(CC, 0), (SSSP, 0), (SSSP, 5002), (WSSSP, 5002)], expect_ragged)


def expect_tiny(g, app, ref):
    assert g.nv // 16 == 0 and ref.pull.all()
    if ref.start == 12 and app != CC:
        assert ref.iters == 1 and ref.active.tolist() == [0]


_case("tiny_nv", tiny, [(CC, 0), (SSSP, 0), (SSSP, 12), (WSSSP, 0), (WSSSP, 12)], expect_tiny)


def expect_sink(g, app, ref):
    assert O.out_degree(g.nv, g.src)[999] == 0
    assert ref.iters == 1 and ref.active.tolist() == [0] and ref.pull.tolist() == [0]


_case("sink_start", sink_start, [(SSSP, 999), (WSSSP, 999)], expect_sink)

CASE_RUNS = [(name, app, start) for name, (_, runs, _) in CASES.items() for app, start in runs]


def case_run_id(r):
    return "%s-%s-%d" % r


# ---- references ----------------------------------------------------------------------------------------------------

_OAPP = {CC: O.APP_CC, SSSP: O.APP_SSSP}


class Ref:
    """Labels L_0..L_n (L_n the fixpoint, n = iters), active[k] = |L_{k+1} != L_k|, pull[k], ftype[k] on one rank."""

    def __init__(self, labels, active, pull, ftype, start):
        self.labels, self.active, self.pull, self.ftype, self.start = labels, active, pull, ftype, start
        self.iters = len(active)


def init_labels(app, nv, start):
    if app == WSSSP:
        lab = np.full(nv, W.INF, np.uint32)
        if start < nv:
            lab[start] = 0
        return lab
    return O.label_init(_OAPP[app], nv, start)


def label_pull(app, row_end, src, weight, lab):
    if app == WSSSP:
        return W.label_pull(row_end, src, weight, lab)[0]
    return O.label_pull(_OAPP[app], row_end, src, lab)[0]


def frontier_rule(nv, first_count, active):
    """(pull, ftype) of each iteration on one rank, from the size of the frontier each one starts from."""
    before = np.concatenate([[first_count], active[:-1]]).astype(np.uint64)
    pull = (before > nv // 16).astype(np.int32)
    ftype = np.where(np.asarray(active, np.uint64) >= cap(nv), O.DENSE_BITMAP, O.SPARSE_QUEUE).astype(np.uint32)
    return pull, ftype


def jacobi(app, row_end, src, weight, lab0, first_count, start=0, max_iters=100000):
    """Iterate label_pull from lab0 up to and including the first iteration that changes nothing.  first_count: size
    of the frontier the first iteration starts from (nv after init for CC or after set_values, 1 for SSSP)."""
    labels = [np.ascontiguousarray(lab0, np.uint32)]
    active = []
    for _ in range(max_iters):
        nxt = label_pull(app, row_end, src, weight, labels[-1])
        active.append(int(np.count_nonzero(nxt != labels[-1])))
        labels.append(nxt)
        if active[-1] == 0:
            break
    active = np.array(active, np.uint64)
    pull, ftype = frontier_rule(len(row_end), first_count, active)
    return Ref(labels, active, pull, ftype, start)


def reference(app, row_end, src, weight, start):
    nv = len(row_end)
    first = nv if app == CC else int(start < nv)
    return jacobi(app, row_end, src, weight, init_labels(app, nv, start), first, start)


def oracle_run(app, row_end, src, weight, start):
    if app == WSSSP:
        return W.label_run(row_end, src, weight, P=1, start=start)
    return O.label_run(_OAPP[app], row_end, src, P=1, start=start)


def assert_jacobi_is_the_oracle(app, row_end, src, weight, start):
    ref = reference(app, row_end, src, weight, start)
    orc = oracle_run(app, row_end, src, weight, start)
    assert ref.iters == orc["iters"]
    assert np.array_equal(ref.labels[-1], orc["labels"])
    assert np.array_equal(ref.active, orc["active"])
    assert np.array_equal(ref.pull, orc["pull"])
    assert np.array_equal(ref.ftype, orc["ftype"][:, 0])
    return ref


def fixture_runs():
    """The fixtures of the GPU stepping test besides the designed cases: ALL_SMALL, RMAT-14/16 (name, builder, runs)."""
    out = []
    for name in sorted(ALL_SMALL):
        def build(name=name):
            row_end, src = ALL_SMALL[name]()
            return row_end, src, case_weights(src, 7)
        nv = len(ALL_SMALL[name]()[0])
        out.append((name, build, [(CC, 0), (SSSP, 0), (SSSP, nv - 1), (WSSSP, 0)]))
    for scale in (14, 16):
        def build_sym(scale=scale):
            row_end, src = symmetrize(*rmat(scale, ef=8))
            return row_end, src, case_weights(src, 3)

        def build_dir(scale=scale):
            row_end, src = rmat(scale)
            return row_end, src, case_weights(src, 3)
        out.append(("rmat%d_sym" % scale, build_sym, [(CC, 0)]))
        out.append(("rmat%d" % scale, build_dir, [(SSSP, 0), (SSSP, 12345), (WSSSP, 0)]))
    return out


FIXTURES = {name: (build, runs) for name, build, runs in fixture_runs()}
FIXTURE_RUNS = [(name, app, start) for name, (_, runs) in FIXTURES.items() for app, start in runs]


def build_run(name):
    """(row_end, src, weight, graph or None) of a designed case or a fixture."""
    if name in CASES:
        g = CASES[name][0]()
        return g.row_end, g.src, g.weight, g
    row_end, src, w = FIXTURES[name][0]()
    return row_end, src, w, None


# ---- tests ---------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("run", CASE_RUNS, ids=case_run_id)
def test_case_hits_its_boundary(run):
    name, app, start = run
    row_end, src, w, g = build_run(name)
    ref = assert_jacobi_is_the_oracle(app, row_end, src, w, start)
    CASES[name][2](g, app, ref)


@pytest.mark.parametrize("run", FIXTURE_RUNS, ids=case_run_id)
def test_jacobi_sequence_is_the_oracle_run(run):
    name, app, start = run
    row_end, src, w, _ = build_run(name)
    assert_jacobi_is_the_oracle(app, row_end, src, w, start)


def test_frontier_rule_at_its_edges():
    nv = NV
    c = cap(nv)
    pull, ftype = frontier_rule(nv, 1, np.array([nv // 16, nv // 16 + 1, c - 1, c, 0], np.uint64))
    assert pull.tolist() == [0, 0, 1, 1, 1]
    assert ftype.tolist() == [O.SPARSE_QUEUE, O.SPARSE_QUEUE, O.SPARSE_QUEUE, O.DENSE_BITMAP, O.SPARSE_QUEUE]
    assert cap(nv) == 4195 and cap(1) == 100


def test_restart_from_a_checkpoint_is_the_rest_of_the_run():
    """A restart from L_k with every vertex active (what set_values installs) pulls once and then follows the same
    labels: label_pull^j(L_k) = L_{k+j}, so the fixpoint is the uninterrupted one."""
    row_end, src, w, _ = build_run("rmat14")
    for app in (SSSP, WSSSP):
        ref = reference(app, row_end, src, w, 0)
        for k in (1, ref.iters // 2):
            again = jacobi(app, row_end, src, w, ref.labels[k], len(row_end))
            assert again.pull[0] == 1
            for j in range(again.iters):
                assert np.array_equal(again.labels[j], ref.labels[min(k + j, ref.iters)])
            assert np.array_equal(again.labels[-1], ref.labels[-1])
