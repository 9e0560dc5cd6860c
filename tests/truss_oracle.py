"""ctypes/numpy front-end of tests/truss_oracle.c, the CPU oracle of the k-truss decomposition (test infrastructure
only), and the generators of inputs whose truss numbers are known in closed form.

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

_SRC = os.path.join(os.path.dirname(os.path.abspath(__file__)), "truss_oracle.c")
_CFLAGS = ["-O3", "-march=x86-64-v3", "-fopenmp", "-fPIC", "-Wall", "-Wextra", "-std=gnu11", "-shared"]
_lib = None


def _p(a):
    return a.ctypes.data_as(C.c_void_p) if a is not None and len(a) else None


def build():
    """Path of the compiled library, building it if this digest of the source has not been built yet."""
    with open(_SRC, "rb") as f:
        digest = hashlib.sha256(f.read() + " ".join(_CFLAGS).encode()).hexdigest()[:16]
    cache = os.path.join(tempfile.gettempdir(), "luxb_truss_oracle_%d" % os.getuid())
    os.makedirs(cache, exist_ok=True)
    so = os.path.join(cache, "libtruss_oracle_%s.so" % digest)
    if not os.path.exists(so):
        tmp = "%s.tmp.%d" % (so, os.getpid())
        subprocess.check_call(["gcc"] + _CFLAGS + ["-o", tmp, _SRC])
        os.replace(tmp, so)  # atomic: concurrent ranks never load a half-written library
    return so


def lib():
    global _lib
    if _lib is None:
        L = C.CDLL(build())
        L.tro_num_edges.restype = C.c_int64
        L.tro_run.restype = C.c_int
        L.tro_check.restype = C.c_int64
        _lib = L
    return _lib


def _csc_args(row_end, src):
    return np.ascontiguousarray(row_end, np.uint64), np.ascontiguousarray(src, np.uint32)


def _num_edges(row_end, src):
    m = lib().tro_num_edges(C.c_uint32(len(row_end)), _p(row_end), _p(src))
    if m < 0:
        raise ValueError("truss oracle: a source id is >= nv, m >= 2^32, or out of memory (%d)" % m)
    return int(m)


def run(row_end, src):
    """k-truss decomposition of the CSC read as an undirected simple graph.  Returns dict(lo, hi = u32 [m] the edges in
    ascending (lo, hi) order, support = u32 [m], truss = u32 [m] by the Wang-Cheng bucket peel, truss_sync = u32 [m] by
    the level-synchronous schedule, vertex = u32 [nv] the largest truss number at each vertex, kmax, rounds, levels,
    trace_active = u64 [rounds] |F| of every round, trace_k = i32 [rounds] its k, max_frontier = largest |F|, m,
    seconds = wall time of the oracle)."""
    row_end, src = _csc_args(row_end, src)
    nv = len(row_end)
    t0 = time.perf_counter()
    m = _num_edges(row_end, src)
    lo, hi, sup, tau, tau_sync = (np.zeros(m, np.uint32) for _ in range(5))
    tv = np.zeros(nv, np.uint32)
    tf, tk = np.zeros(m + 1, np.uint64), np.zeros(m + 1, np.uint32)
    stats = np.zeros(5, np.uint64)
    rc = lib().tro_run(C.c_uint32(nv), _p(row_end), _p(src), _p(lo), _p(hi), _p(sup), _p(tau), _p(tau_sync), _p(tv), _p(tf), _p(tk),
                       _p(stats))
    dt = time.perf_counter() - t0
    if rc != 0:
        raise ValueError("truss oracle failed (%d)" % rc)
    rounds = int(stats[1])
    return dict(lo=lo, hi=hi, support=sup, truss=tau, truss_sync=tau_sync, vertex=tv, kmax=int(stats[3]), rounds=rounds,
                levels=int(stats[2]), trace_active=tf[:rounds].copy(), trace_k=tk[:rounds].astype(np.int32),
                max_frontier=int(stats[4]), m=int(stats[0]), seconds=dt)


def check(row_end, src, truss):
    """(number of edges that fail the truss check under `truss` (u32 [m], edge order of run()), bool [m] which ones)."""
    row_end, src = _csc_args(row_end, src)
    truss = np.ascontiguousarray(truss, np.uint32)
    bad = np.zeros(len(truss), np.uint8)
    n = lib().tro_check(C.c_uint32(len(row_end)), _p(row_end), _p(src), _p(truss), _p(bad))
    if n < 0:
        raise ValueError("truss oracle: a source id is >= nv, or out of memory (%d)" % n)
    return int(n), bad.astype(bool)


# ---- exact inputs: (row_end, src, truss) with the truss number of every edge in closed form ---------------------------
def _csc(n, a, b, tau):
    """Simple edges (a[i], b[i]) with truss numbers tau[i], stored once each as a -> b; truss in (lo, hi) order."""
    a, b = np.asarray(a, np.int64), np.asarray(b, np.int64)
    row_end, src = O.edges_to_csc(n, a, b)
    order = np.lexsort((np.maximum(a, b), np.minimum(a, b)))
    return row_end, src, np.asarray(np.broadcast_to(tau, a.shape), np.uint32)[order]


def complete(n):
    """K_n: every τ = n, every support n - 2, one round."""
    a, b = np.triu_indices(n, 1)
    return _csc(n, a, b, n)


def clique_result(n):
    """What run() returns for K_n (stored as complete(n) is, or any variant of it), in closed form: the oracle's sequential
    peels take minutes on K_2048."""
    lo, hi = (x.astype(np.uint32) for x in np.triu_indices(n, 1))
    m = len(lo)
    return dict(lo=lo, hi=hi, support=np.full(m, n - 2, np.uint32), truss=np.full(m, n, np.uint32), vertex=np.full(n, n, np.uint32),
                kmax=n, rounds=1, m=m, trace_active=np.array([m], np.uint64), trace_k=np.array([n], np.int32))


def cliques(j):
    """Disjoint cliques K_3 .. K_j: τ = c on every edge of K_c."""
    a, b, t, at = [], [], [], 0
    for c in range(3, j + 1):
        i, k = np.triu_indices(c, 1)
        a.append(at + i)
        b.append(at + k)
        t.append(np.full(len(i), c))
        at += c
    return _csc(at, np.concatenate(a), np.concatenate(b), np.concatenate(t))


def book(n):
    """The book B_n: spine {0, 1} and n pages 2 .. n + 1 joined to both: every τ = 3.  The 2n page edges go in the
    first round (support 1), each page's lower edge lowering the spine once (n decrements in one round); the spine, at
    support 0, in the second: trace [2n, 1]."""
    p = 2 + np.arange(n)
    return _csc(n + 2, np.concatenate([[0], np.zeros(n, np.int64), np.ones(n, np.int64)]), np.concatenate([[1], p, p]), 3)


def wheel(rim):
    """Hub 0 joined to a cycle 1 .. rim (rim >= 5): every τ = 3; trace [rim, rim] (the rim edges at support 1, then
    the spokes, lowered twice each, at support 0)."""
    r = np.arange(1, rim + 1)
    return _csc(rim + 1, np.concatenate([np.zeros(rim, np.int64), r]), np.concatenate([r, np.roll(r, -1)]), 3)


def complete_bipartite(p, q):
    """K_{p,q}: no triangle, every τ = 2, one round."""
    return _csc(p + q, np.repeat(np.arange(p), q), p + np.tile(np.arange(q), p), 2)


def cycle(n):
    """C_n (n >= 4): every τ = 2, one round."""
    a = np.arange(n)
    return _csc(n, a, (a + 1) % n, 2)


def grid(r, c):
    """r x c grid: every τ = 2, one round."""
    ids = np.arange(r * c).reshape(r, c)
    a = np.concatenate([ids[:, :-1].ravel(), ids[:-1, :].ravel()])
    b = np.concatenate([ids[:, 1:].ravel(), ids[1:, :].ravel()])
    return _csc(r * c, a, b, 2)


def tube(L, width=6):
    """The triangulated tube: L rings (i, j), j mod width, each a cycle, ring i joined to ring i + 1 by (i, j)-(i+1, j)
    and (i, j)-(i+1, j+1): every τ = 3.  The boundary rings' edges lie in one triangle, every other edge in two; the
    peel eats the tube from both ends, exactly L rounds at k = 3."""
    ids = np.arange(L * width).reshape(L, width)
    nxt = np.roll(ids, -1, axis=1)
    a = np.concatenate([ids.ravel(), ids[:-1].ravel(), ids[:-1].ravel()])
    b = np.concatenate([nxt.ravel(), ids[1:].ravel(), nxt[1:].ravel()])
    return _csc(L * width, a, b, 3)


def no_edges(n=17):
    """n vertices, self-loops only: m = 0, no round, kmax 0."""
    v = np.arange(0, n, 3)
    return _csc(n, v, v, 2)[:2] + (np.zeros(0, np.uint32),)


CLOSED_FORMS = {
    "k48": lambda: complete(48),
    "cliques": lambda: cliques(30),
    "book": lambda: book(1 << 17),
    "wheel": lambda: wheel(1000),
    "k_30_45": lambda: complete_bipartite(30, 45),
    "cycle": lambda: cycle(1000),
    "grid": lambda: grid(40, 60),
    "tube": lambda: tube(3000),
    "no_edges": lambda: no_edges(),
}
