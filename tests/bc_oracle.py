"""ctypes/numpy front-end of tests/bc_oracle.c, the CPU oracle of betweenness centrality (test infrastructure only),
and the generator of exact BC inputs (`forest`).

The library is compiled with gcc on first use into a per-user cache directory keyed by the digest of the C source (the
source tree is never written)."""
import ctypes as C
import hashlib
import os
import subprocess
import tempfile

import numpy as np

import oracle as O

_SRC = os.path.join(os.path.dirname(os.path.abspath(__file__)), "bc_oracle.c")
_CFLAGS = ["-O3", "-march=x86-64-v3", "-fopenmp", "-fPIC", "-ffp-contract=off", "-Wall", "-Wextra", "-std=gnu11", "-shared"]
_lib = None


def _p(a):
    return a.ctypes.data_as(C.c_void_p) if a is not None else None


def build():
    """Path of the compiled library, building it if this digest of the source has not been built yet."""
    with open(_SRC, "rb") as f:
        digest = hashlib.sha256(f.read() + " ".join(_CFLAGS).encode()).hexdigest()[:16]
    cache = os.path.join(tempfile.gettempdir(), "luxb_bc_oracle_%d" % os.getuid())
    os.makedirs(cache, exist_ok=True)
    so = os.path.join(cache, "libbc_oracle_%s.so" % digest)
    if not os.path.exists(so):
        tmp = "%s.tmp.%d" % (so, os.getpid())
        subprocess.check_call(["gcc"] + _CFLAGS + ["-o", tmp, _SRC, "-lm"])
        os.replace(tmp, so)  # atomic: concurrent ranks never load a half-written library
    return so


def lib():
    global _lib
    if _lib is None:
        L = C.CDLL(build())
        L.bco_run.restype = C.c_int
        _lib = L
    return _lib


def run(row_end, src, sources):
    """Brandes from `sources` in order.  Returns dict(scores f64 [nv] (sum of delta_s(v) over s != v), lev / sigma / delta
    of the last source, levels = number of BFS levels of every source)."""
    row_end = np.ascontiguousarray(row_end, np.uint64)
    src = np.ascontiguousarray(src, np.uint32)
    sources = np.ascontiguousarray(np.asarray(sources).reshape(-1), np.uint32)
    nv = len(row_end)
    scores = np.zeros(nv, np.float64)
    lev = np.full(nv, nv, np.uint32)
    sigma = np.zeros(nv, np.float64)
    delta = np.zeros(nv, np.float64)
    levels = np.zeros(max(len(sources), 1), np.uint32)
    rc = lib().bco_run(C.c_uint32(nv), C.c_uint64(len(src)), _p(row_end), _p(src) if len(src) else None, _p(sources),
                       C.c_int(len(sources)), _p(scores), _p(lev), _p(sigma), _p(delta), _p(levels))
    if rc != 0:
        raise ValueError("bc oracle: a source is >= nv, or out of memory")
    return dict(scores=scores, lev=lev, sigma=sigma, delta=delta, levels=levels[:len(sources)].copy())


def source_state(row_end, src, s):
    """(lev, sigma, delta) of the single source s."""
    r = run(row_end, src, [s])
    return r["lev"], r["sigma"], r["delta"]


def scores(row_end, src, sources=None):
    """BC scores over `sources` (None: every vertex, exact BC)."""
    if sources is None:
        sources = np.arange(len(row_end), dtype=np.uint32)
    return run(row_end, src, sources)["scores"]


# ---- exact inputs --------------------------------------------------------------------------------------------------
class Forest:
    """A forest in which every non-root vertex has exactly one parent, on the previous level.  Tree edges appear 1, 2 or
    4 times; extra edges join a vertex only to a vertex of its own level or a shallower one of the same tree (never
    matching the level filter, never shortening a path).  From the roots every sigma is a power of two and every score
    is an integer, the number of descendants, so every summation order is exact."""

    def __init__(self, seed):
        self.rng = np.random.default_rng(seed)
        self.parent, self.level, self.tree, self.mult, self.log_sigma = [], [], [], [], []
        self.roots = []
        self.extra_src, self.extra_dst = [], []

    def add(self, parent, mult=1):
        v = len(self.parent)
        if parent < 0:
            self.parent.append(-1); self.level.append(0); self.tree.append(len(self.roots)); self.mult.append(0)
            self.log_sigma.append(0)
            self.roots.append(v)
        else:
            self.parent.append(parent); self.level.append(self.level[parent] + 1); self.tree.append(self.tree[parent])
            self.mult.append(mult); self.log_sigma.append(self.log_sigma[parent] + {1: 0, 2: 1, 4: 2}[mult])
        return v

    def rand_mult(self, parent, cap=40):
        m = int(self.rng.choice([1, 1, 1, 2, 4]))
        return 1 if self.log_sigma[parent] + 2 > cap else m

    def extra(self, x, y, times=1):
        """x -> y, repeated `times`, with y on x's level or shallower, in x's tree."""
        assert self.tree[x] == self.tree[y] and self.level[y] <= self.level[x]
        self.extra_src += [x] * times
        self.extra_dst += [y] * times

    def csc(self, isolated=0, shuffle=True):
        """dict(row_end, src, roots, descendants, scores = BC from the roots, level, log_sigma, tree) with the vertex ids
        shuffled (trees spread over every partition)."""
        n = len(self.parent) + isolated
        parent = np.array(self.parent, np.int64)
        child = np.nonzero(parent >= 0)[0]
        mult = np.array(self.mult, np.int64)[child]
        es = np.concatenate([np.repeat(parent[child], mult), np.array(self.extra_src, np.int64)])
        ed = np.concatenate([np.repeat(child, mult), np.array(self.extra_dst, np.int64)])
        desc = np.zeros(n, np.int64)
        lev = np.array(self.level, np.int64)
        for v in np.argsort(-lev, kind="stable"):
            if parent[v] >= 0:
                desc[parent[v]] += desc[v] + 1
        perm = self.rng.permutation(n) if shuffle else np.arange(n)
        row_end, src = O.edges_to_csc(n, perm[es], perm[ed])
        new_desc = np.zeros(n, np.int64)
        new_desc[perm] = desc
        new_level = np.full(n, n, np.int64)
        new_level[perm[:len(lev)]] = lev
        new_log_sigma = np.zeros(n, np.int64)
        new_log_sigma[perm[:len(lev)]] = self.log_sigma
        roots = perm[np.array(self.roots, np.int64)].astype(np.uint32)
        scores = new_desc.astype(np.float64)
        scores[roots] = 0  # BC from the roots: a source's own dependency is not counted
        return dict(row_end=row_end, src=src, roots=roots, descendants=new_desc.astype(np.float64), scores=scores, level=new_level,
                    log_sigma=new_log_sigma, tree=self._tree_of(perm, n))

    def _tree_of(self, perm, n):
        t = np.full(n, -1, np.int64)
        t[perm[:len(self.tree)]] = self.tree
        return t


def forest(seed=1, hub_children=1 << 17, hub_in=1 << 20, chain_depth=3000, n_random=24, random_size=1500, isolated=100):
    """The exact-input forest: a hub with `hub_children` children (its delta is cut into segments), a vertex with about
    `hub_in` in-edges none of which matches the level filter (its sigma is cut into segments), a chain `chain_depth`
    levels deep, and `n_random` random trees.  Returns Forest.csc()."""
    F = Forest(seed)
    # the hub tree
    r = F.add(-1)
    h = F.add(r, 2)
    y = F.add(r, 1)
    kids = [F.add(h, int(m)) for m in F.rng.choice([1, 2, 4], hub_children)]
    per = max(1, hub_in // max(len(kids), 1))
    for k in kids:
        F.extra(k, y, per)
    F.extra(h, y, 3)   # same level
    F.extra(y, y, 2)   # self-loops
    F.extra(kids[0], r, 1)
    # the chain, with side leaves and back edges
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
            if F.level[y] > F.level[x]:
                x, y = y, x
            F.extra(x, y, int(F.rng.choice([1, 2])))
    return F.csc(isolated=isolated)


def small_forest(seed=3):
    """A few hundred vertices of the same kind (quick tests, several ranks)."""
    return forest(seed=seed, hub_children=300, hub_in=5000, chain_depth=200, n_random=6, random_size=60, isolated=7)
