"""ctypes/numpy front-end of tests/bc_weighted_oracle.c, the CPU oracle of weighted betweenness centrality (test
infrastructure only), and the generator of exact weighted BC inputs (`forest`).

The library is compiled with gcc on first use into a per-user cache directory keyed by the digest of the C source (the
source tree is never written)."""
import ctypes as C
import hashlib
import os
import subprocess
import tempfile

import numpy as np

_SRC = os.path.join(os.path.dirname(os.path.abspath(__file__)), "bc_weighted_oracle.c")
_CFLAGS = ["-O3", "-march=x86-64-v3", "-fopenmp", "-fPIC", "-ffp-contract=off", "-Wall", "-Wextra", "-std=gnu11", "-shared"]
_lib = None

INF = 0xFFFFFFFF  # distance of an unreachable vertex (LUXB_DIST_INF)


def _p(a):
    return a.ctypes.data_as(C.c_void_p) if a is not None else None


def build():
    """Path of the compiled library, building it if this digest of the source has not been built yet."""
    with open(_SRC, "rb") as f:
        digest = hashlib.sha256(f.read() + " ".join(_CFLAGS).encode()).hexdigest()[:16]
    cache = os.path.join(tempfile.gettempdir(), "luxb_bc_weighted_oracle_%d" % os.getuid())
    os.makedirs(cache, exist_ok=True)
    so = os.path.join(cache, "libbc_weighted_oracle_%s.so" % digest)
    if not os.path.exists(so):
        tmp = "%s.tmp.%d" % (so, os.getpid())
        subprocess.check_call(["gcc"] + _CFLAGS + ["-o", tmp, _SRC, "-lm"])
        os.replace(tmp, so)  # atomic: concurrent ranks never load a half-written library
    return so


def lib():
    global _lib
    if _lib is None:
        L = C.CDLL(build())
        L.bwo_run.restype = C.c_int
        _lib = L
    return _lib


def run(row_end, src, weight, sources):
    """Weighted Brandes from `sources` in order.  Returns dict(scores f64 [nv] (sum of delta_s(v) over s != v), dist /
    sigma / delta of the last source, classes = number of distinct distances of every source)."""
    row_end = np.ascontiguousarray(row_end, np.uint64)
    src = np.ascontiguousarray(src, np.uint32)
    weight = np.ascontiguousarray(weight, np.int32)
    assert len(weight) == len(src), "one weight per edge"
    sources = np.ascontiguousarray(np.asarray(sources).reshape(-1), np.uint32)
    nv = len(row_end)
    scores = np.zeros(nv, np.float64)
    dist = np.full(nv, INF, np.uint32)
    sigma = np.zeros(nv, np.float64)
    delta = np.zeros(nv, np.float64)
    classes = np.zeros(max(len(sources), 1), np.uint32)
    rc = lib().bwo_run(C.c_uint32(nv), C.c_uint64(len(src)), _p(row_end), _p(src) if len(src) else None,
                       _p(weight) if len(src) else None, _p(sources), C.c_int(len(sources)), _p(scores), _p(dist), _p(sigma),
                       _p(delta), _p(classes))
    if rc == -2:
        raise ValueError("weighted bc oracle: a weight is < 1 (weighted betweenness centrality needs w >= 1)")
    if rc != 0:
        raise ValueError("weighted bc oracle: a source is >= nv, or out of memory")
    return dict(scores=scores, dist=dist, sigma=sigma, delta=delta, classes=classes[:len(sources)].copy())


def source_state(row_end, src, weight, s):
    """(dist, sigma, delta) of the single source s."""
    r = run(row_end, src, weight, [s])
    return r["dist"], r["sigma"], r["delta"]


def scores(row_end, src, weight, sources=None):
    """Weighted BC scores over `sources` (None: every vertex, exact BC)."""
    if sources is None:
        sources = np.arange(len(row_end), dtype=np.uint32)
    return run(row_end, src, weight, sources)["scores"]


def edges_to_csc(nv, esrc, edst, ew):
    """(row_end, src, weight) of a weighted edge list in canonical (dst, src) order (ties keep the list order)."""
    esrc, edst, ew = np.asarray(esrc, np.int64), np.asarray(edst, np.int64), np.asarray(ew, np.int64)
    order = np.lexsort((esrc, edst))
    row_end = np.cumsum(np.bincount(edst, minlength=nv)).astype(np.uint64)
    return row_end, esrc[order].astype(np.uint32), ew[order].astype(np.int32)


def csc_dst(row_end):
    """Destination of every CSC edge."""
    return np.repeat(np.arange(len(row_end), dtype=np.int64), np.diff(np.concatenate([[0], row_end]).astype(np.int64)))


# ---- exact inputs --------------------------------------------------------------------------------------------------
class Forest:
    """A weighted forest: every non-root vertex has exactly one parent, its tree edge has a weight in [1, 255] and appears
    1, 2 or 4 times at that weight.  Extra edges x -> y (same tree) have D[x] + w > D[y], so they are never tight and
    never shorten a path; they may go to deeper vertices, and near misses have D[x] + w = D[y] + 1.  From the roots the
    tight edges are the tree edges: every sigma is a power of two and every score is the number of descendants, so
    every summation order is exact."""

    def __init__(self, seed):
        self.rng = np.random.default_rng(seed)
        self.parent, self.dist, self.tree, self.mult, self.wt, self.log_sigma = [], [], [], [], [], []
        self.roots = []
        self.extra_src, self.extra_dst, self.extra_w = [], [], []

    def add(self, parent, mult=1, w=None):
        v = len(self.parent)
        if parent < 0:
            self.parent.append(-1); self.dist.append(0); self.tree.append(len(self.roots)); self.mult.append(0); self.wt.append(0)
            self.log_sigma.append(0)
            self.roots.append(v)
        else:
            w = int(self.rng.integers(1, 256)) if w is None else w
            self.parent.append(parent); self.dist.append(self.dist[parent] + w); self.tree.append(self.tree[parent])
            self.mult.append(mult); self.wt.append(w); self.log_sigma.append(self.log_sigma[parent] + {1: 0, 2: 1, 4: 2}[mult])
        return v

    def rand_mult(self, parent, cap=40):
        m = int(self.rng.choice([1, 1, 1, 2, 4]))
        return 1 if self.log_sigma[parent] + 2 > cap else m

    def extra(self, x, y, times=1, slack=None):
        """x -> y, repeated `times`, in x's tree, with D[x] + w = D[y] + 1 + slack (slack >= 0 random if None)."""
        assert self.tree[x] == self.tree[y]
        slack = int(self.rng.integers(0, 300)) if slack is None else slack
        w = max(1, self.dist[y] - self.dist[x] + 1 + slack)
        assert self.dist[x] + w > self.dist[y]
        self.extra_src += [x] * times
        self.extra_dst += [y] * times
        self.extra_w += [w] * times

    def csc(self, isolated=0, shuffle=True):
        """dict(row_end, src, weight, roots, descendants, scores = BC from the roots, dist, log_sigma, tree) with the vertex
        ids shuffled (trees spread over every partition)."""
        n = len(self.parent) + isolated
        parent = np.array(self.parent, np.int64)
        child = np.nonzero(parent >= 0)[0]
        mult = np.array(self.mult, np.int64)[child]
        es = np.concatenate([np.repeat(parent[child], mult), np.array(self.extra_src, np.int64)])
        ed = np.concatenate([np.repeat(child, mult), np.array(self.extra_dst, np.int64)])
        ew = np.concatenate([np.repeat(np.array(self.wt, np.int64)[child], mult), np.array(self.extra_w, np.int64)])
        dist = np.array(self.dist, np.int64)
        desc = np.zeros(n, np.int64)
        for v in np.argsort(-dist, kind="stable"):
            if parent[v] >= 0:
                desc[parent[v]] += desc[v] + 1
        perm = self.rng.permutation(n) if shuffle else np.arange(n)
        row_end, src, weight = edges_to_csc(n, perm[es], perm[ed], ew)
        new_desc = np.zeros(n, np.int64)
        new_desc[perm] = desc
        new_dist = np.full(n, INF, np.int64)
        new_dist[perm[:len(dist)]] = dist
        new_log_sigma = np.zeros(n, np.int64)
        new_log_sigma[perm[:len(dist)]] = self.log_sigma
        tree = np.full(n, -1, np.int64)
        tree[perm[:len(self.tree)]] = self.tree
        roots = perm[np.array(self.roots, np.int64)].astype(np.uint32)
        scores = new_desc.astype(np.float64)
        scores[roots] = 0  # BC from the roots: a source's own dependency is not counted
        return dict(row_end=row_end, src=src, weight=weight, roots=roots, descendants=new_desc.astype(np.float64), scores=scores,
                    dist=new_dist, log_sigma=new_log_sigma, tree=tree)


def forest(seed=1, hub_children=1 << 17, hub_in=1 << 20, chain_depth=1500, n_random=24, random_size=1500, isolated=100):
    """The exact weighted forest: a hub with `hub_children` children (its delta is cut into segments), a vertex with about
    `hub_in` non-tight in-edges (its sigma is cut into segments), a chain of `chain_depth` vertices (as many distinct
    distances) and `n_random` random trees.  Returns Forest.csc()."""
    F = Forest(seed)
    # the hub tree
    r = F.add(-1)
    h = F.add(r, 2)
    y = F.add(r, 1)
    kids = [F.add(h, int(m)) for m in F.rng.choice([1, 2, 4], hub_children)]
    per = max(1, hub_in // max(len(kids), 1))
    for k in kids:
        F.extra(k, y, per)
    F.extra(h, y, 3)          # no shorter, from a sibling
    F.extra(y, y, 2)          # self-loops
    F.extra(r, kids[0], 2, slack=0)  # a near miss into a deeper vertex, twice
    F.extra(kids[0], r, 1)
    # the chain, with side leaves, back edges and near misses forward
    r = F.add(-1)
    prev = r
    path = [r]
    for d in range(1, chain_depth):
        v = F.add(prev, 2 if d % 150 == 0 else 1)
        path.append(v)
        if d % 7 == 0:
            F.add(v, F.rand_mult(v))
        if d % 11 == 0:
            F.extra(v, path[int(F.rng.integers(0, d + 1))], 1)
        if d % 13 == 0 and d >= 3:
            F.extra(path[d - 3], v, 1, slack=0)
        prev = v
    # random trees
    for _ in range(n_random):
        r = F.add(-1)
        members = [r]
        size = int(F.rng.integers(1, random_size))
        for _ in range(size):
            p = members[int(F.rng.integers(0, len(members)))]
            members.append(F.add(p, F.rand_mult(p)))
        for _ in range(size // 2):
            x = members[int(F.rng.integers(0, len(members)))]
            y = members[int(F.rng.integers(0, len(members)))]
            F.extra(x, y, int(F.rng.choice([1, 2])), slack=int(F.rng.choice([0, 0, 5, 100])))
    return F.csc(isolated=isolated)


def small_forest(seed=3):
    """A few hundred vertices of the same kind (quick tests, several ranks)."""
    return forest(seed=seed, hub_children=300, hub_in=5000, chain_depth=200, n_random=6, random_size=60, isolated=7)
