"""ctypes/numpy front-end of tests/weighted_oracle.c, the CPU oracle of weighted SSSP (test infrastructure only).

The library is compiled with gcc on first use into a per-user cache directory keyed by the digest of the C source (the
source tree is never written).  Partition bounds come from the reference partitioner of `oracle` (oracle.partition),
with the same rule as oracle.label_run for a remainder of zero-in-degree vertices."""
import ctypes as C
import hashlib
import os
import subprocess
import tempfile

import numpy as np

import oracle as O

_SRC = os.path.join(os.path.dirname(os.path.abspath(__file__)), "weighted_oracle.c")
_CFLAGS = ["-O3", "-march=x86-64-v3", "-fopenmp", "-fPIC", "-ffp-contract=off", "-Wall", "-Wextra", "-std=gnu11", "-shared"]
_lib = None

INF = 0xFFFFFFFF  # distance of an unreachable vertex (LUXB_DIST_INF)
SPARSE_THRESHOLD = 16


def _p(a):
    return a.ctypes.data_as(C.c_void_p) if a is not None else None


def build():
    """Path of the compiled library, building it if this digest of the source has not been built yet."""
    with open(_SRC, "rb") as f:
        digest = hashlib.sha256(f.read() + " ".join(_CFLAGS).encode()).hexdigest()[:16]
    cache = os.path.join(tempfile.gettempdir(), "luxb_weighted_oracle_%d" % os.getuid())
    os.makedirs(cache, exist_ok=True)
    so = os.path.join(cache, "libweighted_oracle_%s.so" % digest)
    if not os.path.exists(so):
        tmp = "%s.tmp.%d" % (so, os.getpid())
        subprocess.check_call(["gcc"] + _CFLAGS + ["-o", tmp, _SRC, "-lm"])
        os.replace(tmp, so)  # atomic: concurrent ranks never load a half-written library
    return so


def lib():
    global _lib
    if _lib is None:
        L = C.CDLL(build())
        L.wo_rmat_weight.restype = C.c_int32
        L.wo_rmat_weight.argtypes = [C.c_uint64, C.c_uint32, C.c_uint32]
        L.wo_sat_add.restype = C.c_uint32
        L.wo_sat_add.argtypes = [C.c_uint32, C.c_int32]
        L.wo_pull_range.restype = C.c_uint64
        L.wo_check.restype = C.c_uint64
        _lib = L
    return _lib


def _arrays(row_end, src, weight):
    row_end = np.ascontiguousarray(row_end, np.uint64)
    src = np.ascontiguousarray(src, np.uint32)
    weight = np.ascontiguousarray(weight, np.int32)
    assert len(weight) == len(src), "one weight per edge"
    return row_end, src, weight


def rmat_weight(seed, src, dst):
    """Weight of the RMAT edge src -> dst: an int in [1, 255] that depends only on (seed, src, dst)."""
    return lib().wo_rmat_weight(C.c_uint64(seed & (2**64 - 1)), C.c_uint32(src), C.c_uint32(dst))


def rmat_weights(seed, row_end, src):
    """rmat_weight of every edge of a CSC, in CSC order (i32 [ne])."""
    row_end = np.ascontiguousarray(row_end, np.uint64)
    src = np.ascontiguousarray(src, np.uint32)
    w = np.empty(max(len(src), 1), np.int32)[:len(src)]
    lib().wo_rmat_csc_weights(C.c_uint64(seed & (2**64 - 1)), C.c_uint32(len(row_end)), _p(row_end), _p(src), _p(w))
    return w


def sat_add(d, w):
    return lib().wo_sat_add(C.c_uint32(d), C.c_int32(w))


def partitions(row_end, ne, P):
    """(row_left, row_right) of the P partitions: the reference's greedy split; a trailing remainder of zero-in-degree
    vertices becomes a last, edge-free partition (what the product and oracle.label_run do)."""
    nv = len(row_end)
    n, rl, rr, _, _, _ = O.partition(row_end, ne, P)
    if n == P - 1 and (n == 0 or rr[n - 1] < nv - 1):
        rl[n] = 0 if n == 0 else rr[n - 1] + 1
        rr[n] = nv - 1
        n += 1
    if n != P:
        raise ValueError("reference partitioner does not yield P=%d partitions for this graph" % P)
    return rl, rr


def label_run(row_end, src, weight, P=1, start=0, max_iters=10000):
    """Weighted SSSP with the iteration structure of oracle.label_run.
    Returns dict(labels, iters, active[iters], pull[iters], ftype[iters,P])."""
    row_end, src, weight = _arrays(row_end, src, weight)
    nv, ne = len(row_end), len(src)
    rl, rr = partitions(row_end, ne, P)
    lab = np.empty(nv, np.uint32)
    active = np.zeros(max_iters, np.uint64)
    pull = np.zeros(max_iters, np.int32)
    ftype = np.zeros((max_iters, P), np.uint32)
    it = lib().wo_run(C.c_uint32(nv), C.c_uint64(ne), _p(row_end), _p(src), _p(weight), C.c_int(P), _p(rl), _p(rr),
                      C.c_uint32(start), _p(lab), C.c_int(max_iters), _p(active), _p(pull), _p(ftype))
    return dict(labels=lab, iters=it, active=active[:it].copy(), pull=pull[:it].copy(), ftype=ftype[:it].copy())


def label_pull(row_end, src, weight, old):
    """One Jacobi pull sweep over every vertex; returns (new labels, #changed)."""
    row_end, src, weight = _arrays(row_end, src, weight)
    old = np.ascontiguousarray(old, np.uint32)
    new = old.copy()
    changed = lib().wo_pull_range(_p(row_end), _p(src), _p(weight), _p(old), _p(new), C.c_uint32(0), C.c_uint32(len(row_end) - 1))
    return new, changed


def build_push_csr(row_end, src, weight, v_lo, v_hi):
    """CSR-by-source over the edges of destinations [v_lo, v_hi]: (out_end u64[nv], out_dst u32[], out_w i32[])."""
    row_end, src, weight = _arrays(row_end, src, weight)
    nv = len(row_end)
    e_lo = 0 if v_lo == 0 else int(row_end[v_lo - 1])
    n = int(row_end[v_hi]) - e_lo
    out_end = np.empty(nv, np.uint64)
    out_dst = np.empty(max(n, 1), np.uint32)[:n]
    out_w = np.empty(max(n, 1), np.int32)[:n]
    lib().wo_build_push_csr(C.c_uint32(nv), _p(row_end), _p(src), _p(weight), C.c_uint32(v_lo), C.c_uint32(v_hi), _p(out_end),
                            _p(out_dst), _p(out_w))
    return out_end, out_dst, out_w


def label_check(row_end, src, weight, label):
    """Number of in-edges with D[u] != INF and D[v] > sat_add(D[u], w)."""
    row_end, src, weight = _arrays(row_end, src, weight)
    label = np.ascontiguousarray(label, np.uint32)
    return int(lib().wo_check(C.c_uint32(len(row_end)), _p(row_end), _p(src), _p(weight), _p(label)))
