"""ctypes/numpy front-end of tests/tc_oracle.c, the CPU oracle of triangle counting (test infrastructure only), and the
generators of the exact triangle-counting inputs (closed-form counts, no oracle needed) and of the noise variants.

The library is compiled with gcc on first use into a per-user cache directory keyed by the digest of the C source (the
source tree is never written)."""
import ctypes as C
import hashlib
import os
import subprocess
import tempfile
import time

import numpy as np

import oracle as O

_SRC = os.path.join(os.path.dirname(os.path.abspath(__file__)), "tc_oracle.c")
_CFLAGS = ["-O3", "-march=x86-64-v3", "-fopenmp", "-fPIC", "-Wall", "-Wextra", "-std=gnu11", "-shared"]
_lib = None


def _p(a):
    return a.ctypes.data_as(C.c_void_p) if a is not None else None


def build():
    """Path of the compiled library, building it if this digest of the source has not been built yet."""
    with open(_SRC, "rb") as f:
        digest = hashlib.sha256(f.read() + " ".join(_CFLAGS).encode()).hexdigest()[:16]
    cache = os.path.join(tempfile.gettempdir(), "luxb_tc_oracle_%d" % os.getuid())
    os.makedirs(cache, exist_ok=True)
    so = os.path.join(cache, "libtc_oracle_%s.so" % digest)
    if not os.path.exists(so):
        tmp = "%s.tmp.%d" % (so, os.getpid())
        subprocess.check_call(["gcc"] + _CFLAGS + ["-o", tmp, _SRC])
        os.replace(tmp, so)  # atomic: concurrent ranks never load a half-written library
    return so


def lib():
    global _lib
    if _lib is None:
        L = C.CDLL(build())
        L.tco_run.restype = C.c_int
        _lib = L
    return _lib


def run(row_end, src):
    """Triangle counts of the CSC read as an undirected simple graph.  Returns dict(t = u64 [nv] triangles at each
    vertex, total = T, m = undirected simple edges, probes = sum of |N+(v)| over the degree-oriented edges (u, v),
    max_out = largest |N+(u)|, seconds = wall time of the oracle, threads = OpenMP threads it used)."""
    row_end = np.ascontiguousarray(row_end, np.uint64)
    src = np.ascontiguousarray(src, np.uint32)
    nv = len(row_end)
    t = np.zeros(nv, np.uint64)
    stats = np.zeros(5, np.uint64)
    t0 = time.perf_counter()
    rc = lib().tco_run(C.c_uint32(nv), C.c_uint64(len(src)), _p(row_end), _p(src) if len(src) else None, _p(t), _p(stats))
    dt = time.perf_counter() - t0
    if rc != 0:
        raise ValueError("tc oracle: a source id is >= nv, or out of memory (%d)" % rc)
    return dict(t=t, total=int(stats[0]), m=int(stats[1]), probes=int(stats[2]), max_out=int(stats[3]), seconds=dt,
                threads=int(stats[4]))


# ---- exact inputs: (row_end, src, t) with t in closed form -------------------------------------------------------------
def _csc(n, a, b, t):
    row_end, src = O.edges_to_csc(n, np.asarray(a, np.int64), np.asarray(b, np.int64))
    return row_end, src, np.asarray(t, np.uint64)


def complete(n):
    """K_n, every edge stored once (lower id -> higher id): every t = C(n - 1, 2)."""
    a, b = np.triu_indices(n, 1)
    return _csc(n, a, b, np.full(n, (n - 1) * (n - 2) // 2))


def wheel(rim):
    """Wheel: hub 0 joined to a cycle of `rim` vertices 1..rim: t[hub] = rim, every rim vertex 2 (rim >= 4)."""
    r = np.arange(1, rim + 1)
    a = np.concatenate([np.zeros(rim, np.int64), r])
    b = np.concatenate([r, np.roll(r, -1)])
    return _csc(rim + 1, a, b, np.concatenate([[rim], np.full(rim, 2)]))


def windmill(k):
    """Windmill (friendship graph): k triangles sharing centre 0: t[0] = k, every other vertex 1."""
    x = np.arange(k) * 2 + 1
    a = np.concatenate([np.zeros(k, np.int64), np.zeros(k, np.int64), x])
    b = np.concatenate([x, x + 1, x + 1])
    return _csc(2 * k + 1, a, b, np.concatenate([[k], np.ones(2 * k)]))


def complete_bipartite(p, q):
    """K_{p,q}: p * q edges and no triangle."""
    a = np.repeat(np.arange(p), q)
    b = p + np.tile(np.arange(q), p)
    return _csc(p + q, a, b, np.zeros(p + q))


def over_budget(B, H):
    """A graph whose largest out-lists exceed B entries by construction.  Vertex 0 is adjacent to B + 4 heavy vertices;
    every heavy vertex is joined to the same B + 8 leaves; H disjoint heavy-heavy edges (a matching, so no triangle lies
    among the heavies).  Heavies have degree >= B + 9 and rank above vertex 0, whose degree B + 4 ties with the leaves'
    and wins on id: |N+(0)| = B + 4, and every leaf's out-list (the B + 4 heavies) exceeds B as well.  Each matching
    edge closes B + 9 triangles (with 0 and with every leaf): t[0] = t[leaf] = H, t[matched heavy] = B + 9, other
    heavies 0, T = H (B + 9)."""
    nh, nl = B + 4, B + 8
    assert 2 * H <= nh
    heavy = 1 + np.arange(nh)
    leaf = 1 + nh + np.arange(nl)
    a = np.concatenate([np.zeros(nh, np.int64), np.repeat(heavy, nl), heavy[0:2 * H:2]])
    b = np.concatenate([heavy, np.tile(leaf, nh), heavy[1:2 * H:2]])
    t = np.zeros(1 + nh + nl, np.int64)
    t[0] = H
    t[leaf] = H
    t[heavy[:2 * H]] = B + 9
    return _csc(1 + nh + nl, a, b, t)


# ---- noise: the same undirected simple graph stored differently ------------------------------------------------------
def edges_of(row_end, src):
    dst = np.repeat(np.arange(len(row_end), dtype=np.int64), np.diff(np.concatenate([[0], row_end]).astype(np.int64)))
    return src.astype(np.int64), dst


def variant(row_end, src, kind, seed=0):
    """The graph of (row_end, src) stored another way, with the same triangles: "reversed" (every edge flipped),
    "both" (both directions), "mult" (each edge 1, 2 or 4 times, at random), "loops" (plus a self-loop at a third of the
    vertices, some repeated), "mixed" (each edge once in a random direction)."""
    nv = len(row_end)
    a, b = edges_of(row_end, src)
    rng = np.random.default_rng(seed)
    if kind == "reversed":
        a, b = b, a
    elif kind == "both":
        a, b = np.concatenate([a, b]), np.concatenate([b, a])
    elif kind == "mult":
        r = rng.choice([1, 2, 4], len(a))
        a, b = np.repeat(a, r), np.repeat(b, r)
    elif kind == "loops":
        v = rng.choice(nv, max(nv // 3, 1), replace=True)
        a, b = np.concatenate([a, v]), np.concatenate([b, v])
    elif kind == "mixed":
        f = rng.random(len(a)) < 0.5
        a, b = np.where(f, b, a), np.where(f, a, b)
    else:
        raise ValueError(kind)
    return O.edges_to_csc(nv, a, b)


VARIANTS = ("reversed", "both", "mult", "loops", "mixed")
