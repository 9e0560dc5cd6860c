"""ctypes/numpy front-end of tests/kcore_oracle.c, the CPU oracle of the k-core decomposition (test infrastructure
only), and the generators of inputs whose core numbers are known in closed form.

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

_SRC = os.path.join(os.path.dirname(os.path.abspath(__file__)), "kcore_oracle.c")
_CFLAGS = ["-O3", "-march=x86-64-v3", "-fopenmp", "-fPIC", "-Wall", "-Wextra", "-std=gnu11", "-shared"]
_lib = None


def _p(a):
    return a.ctypes.data_as(C.c_void_p) if a is not None and len(a) else None


def build():
    """Path of the compiled library, building it if this digest of the source has not been built yet."""
    with open(_SRC, "rb") as f:
        digest = hashlib.sha256(f.read() + " ".join(_CFLAGS).encode()).hexdigest()[:16]
    cache = os.path.join(tempfile.gettempdir(), "luxb_kcore_oracle_%d" % os.getuid())
    os.makedirs(cache, exist_ok=True)
    so = os.path.join(cache, "libkcore_oracle_%s.so" % digest)
    if not os.path.exists(so):
        tmp = "%s.tmp.%d" % (so, os.getpid())
        subprocess.check_call(["gcc"] + _CFLAGS + ["-o", tmp, _SRC])
        os.replace(tmp, so)  # atomic: concurrent ranks never load a half-written library
    return so


def lib():
    global _lib
    if _lib is None:
        L = C.CDLL(build())
        L.kco_run.restype = C.c_int
        L.kco_check.restype = C.c_int64
        _lib = L
    return _lib


def _csc_args(row_end, src):
    return np.ascontiguousarray(row_end, np.uint64), np.ascontiguousarray(src, np.uint32)


def run(row_end, src):
    """Core numbers of the CSC read as an undirected simple graph.  Returns dict(core = u32 [nv] by Batagelj-Zaversnik,
    core_sync = u32 [nv] by the level-synchronous schedule, degeneracy, rounds, levels, trace_active = u64 [rounds] |F|
    of every round, trace_k = i32 [rounds] its k, max_frontier = largest |F|, m = undirected simple edges, seconds =
    wall time of the oracle)."""
    row_end, src = _csc_args(row_end, src)
    nv = len(row_end)
    core, core_sync = np.zeros(nv, np.uint32), np.zeros(nv, np.uint32)
    tf, tk = np.zeros(nv + 1, np.uint64), np.zeros(nv + 1, np.uint32)
    stats = np.zeros(5, np.uint64)
    t0 = time.perf_counter()
    rc = lib().kco_run(C.c_uint32(nv), _p(row_end), _p(src), _p(core), _p(core_sync), _p(tf), _p(tk), _p(stats))
    dt = time.perf_counter() - t0
    if rc != 0:
        raise ValueError("kcore oracle: a source id is >= nv, or out of memory (%d)" % rc)
    rounds = int(stats[1])
    return dict(core=core, core_sync=core_sync, degeneracy=int(stats[3]), rounds=rounds, levels=int(stats[2]),
                trace_active=tf[:rounds].copy(), trace_k=tk[:rounds].astype(np.int32), max_frontier=int(stats[4]),
                m=int(stats[0]), seconds=dt)


def check(row_end, src, core):
    """(number of vertices that are not a fixpoint of the h-index operator under `core`, bool [nv] which ones)."""
    row_end, src = _csc_args(row_end, src)
    nv = len(row_end)
    core = np.ascontiguousarray(core, np.uint32)
    bad = np.zeros(nv, np.uint8)
    n = lib().kco_check(C.c_uint32(nv), _p(row_end), _p(src), _p(core), _p(bad))
    if n < 0:
        raise ValueError("kcore oracle: a source id is >= nv, or out of memory (%d)" % n)
    return int(n), bad.astype(bool)


# ---- exact inputs: (row_end, src, core) with core in closed form -------------------------------------------------------
def _csc(n, a, b, core):
    row_end, src = O.edges_to_csc(n, np.asarray(a, np.int64), np.asarray(b, np.int64))
    return row_end, src, np.asarray(core, np.uint32)


def complete(n):
    """K_n, every edge stored once: every core n - 1."""
    a, b = np.triu_indices(n, 1)
    return _csc(n, a, b, np.full(n, n - 1))


def complete_bipartite(p, q):
    """K_{p,q}: every core min(p, q)."""
    a = np.repeat(np.arange(p), q)
    b = p + np.tile(np.arange(q), p)
    return _csc(p + q, a, b, np.full(p + q, min(p, q)))


def cycle(n):
    """C_n (n >= 3): every core 2."""
    a = np.arange(n)
    return _csc(n, a, (a + 1) % n, np.full(n, 2))


def grid(r, c):
    """r x c grid (r, c >= 2): every core 2."""
    ids = np.arange(r * c).reshape(r, c)
    a = np.concatenate([ids[:, :-1].ravel(), ids[:-1, :].ravel()])
    b = np.concatenate([ids[:, 1:].ravel(), ids[1:, :].ravel()])
    return _csc(r * c, a, b, np.full(r * c, 2))


def star(leaves):
    """Hub 0 and `leaves` leaves: every core 1.  The leaves go in the first round; the hub's degree then crosses 2 -> 1
    under `leaves` decrements at once and it goes in the second."""
    x = np.arange(1, leaves + 1)
    return _csc(leaves + 1, np.zeros(leaves, np.int64), x, np.ones(leaves + 1))


def path(n):
    """Path of n vertices: every core 1; one level, the two ends per round, then the middle vertex ((n + 1) / 2 rounds
    for odd n)."""
    a = np.arange(n - 1)
    return _csc(n, a, a + 1, np.ones(n) if n > 1 else np.zeros(n))


def clique_chain(lo, hi):
    """Cliques K_lo .. K_hi in a row, the last vertex of each joined to the first of the next by one edge: core c - 1 in
    K_c (a bridge adds one to two vertices only, too few for the c-core)."""
    a, b, core, at, prev = [], [], [], 0, None
    for c in range(lo, hi + 1):
        i, j = np.triu_indices(c, 1)
        a.append(at + i)
        b.append(at + j)
        if prev is not None:
            a.append(np.array([prev]))
            b.append(np.array([at]))
        core.append(np.full(c, c - 1))
        prev = at + c - 1
        at += c
    return _csc(at, np.concatenate(a), np.concatenate(b), np.concatenate(core))


def hub_clique(n, leaves):
    """K_n on 0..n-1, a hub n joined to all of it and to `leaves` leaves: hub and clique n (they form K_{n+1}), leaves 1.
    The hub's lists are mostly leaves, dead by the time the hub goes."""
    i, j = np.triu_indices(n, 1)
    x = n + 1 + np.arange(leaves)
    a = np.concatenate([i, np.full(n + leaves, n)])
    b = np.concatenate([j, np.arange(n), x])
    return _csc(n + 1 + leaves, a, b, np.concatenate([np.full(n + 1, n), np.ones(leaves)]))


CLOSED_FORMS = {
    "k64": lambda: complete(64),
    "k_30_45": lambda: complete_bipartite(30, 45),
    "cycle": lambda: cycle(1000),
    "grid": lambda: grid(40, 60),
    "star": lambda: star(1 << 17),
    "path": lambda: path(3001),
    "clique_chain": lambda: clique_chain(2, 200),
    "hub_clique": lambda: hub_clique(101, 1 << 17),
}
