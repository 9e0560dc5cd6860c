"""ctypes binding of include/lux_b200.h (the drop-in C ABI).  One LuxGraph = one rank = one GPU."""
import ctypes as C
import os
import re
import numpy as np

from . import build as _build

APP_PAGERANK, APP_CC, APP_SSSP, APP_COLFILTER, APP_SSSP_WEIGHTED, APP_BC, APP_BC_WEIGHTED, APP_TC, APP_KCORE, APP_TRUSS = 0, 1, 2, 3, 4, 5, 6, 7, 8, 9
DIST_INF = 0xFFFFFFFF  # APP_SSSP_WEIGHTED / APP_BC_WEIGHTED: distance of an unreachable vertex (LUXB_DIST_INF)
EXCHANGE_NCCL, EXCHANGE_P2P, EXCHANGE_P2P_FUSED = 0, 1, 2
DENSE_BITMAP, SPARSE_QUEUE = 0x1234567, 0x7654321
CF_K = 20
MAX_PARTS = 64
UNIQUE_ID_BYTES = 128

_HEADER = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "include", "lux_b200.h")
_lib = None


class LuxError(RuntimeError):
    pass


class _Csc(C.Structure):
    _fields_ = [("nv", C.c_uint32), ("ne", C.c_uint64), ("row_end", C.c_void_p), ("src", C.c_void_p),
                ("weight", C.c_void_p)]


class _Config(C.Structure):
    _fields_ = [("app", C.c_int), ("rank", C.c_int), ("nranks", C.c_int), ("device", C.c_int),
                ("start_vtx", C.c_uint32), ("exchange", C.c_int), ("verbose", C.c_int), ("balanced_split", C.c_int),
                ("zero_copy_edges", C.c_int)]


class Stats(C.Structure):
    _fields_ = [("loop_seconds", C.c_double), ("iterations", C.c_uint64), ("edges_processed", C.c_uint64),
                ("pull_iterations", C.c_uint64), ("kernel_launches", C.c_uint64), ("last_active", C.c_uint64),
                ("last_frontier_type", C.c_uint32), ("dominant_kernel_seconds", C.c_double),
                ("dominant_kernel_launches", C.c_uint64), ("panel_edges", C.c_uint64), ("panel_hubs", C.c_uint32),
                ("panel_blocks", C.c_uint32), ("cold_hub_edges", C.c_uint64), ("cold_hub_segments", C.c_uint32),
                ("tier_blocks", C.c_uint32), ("tier_slots", C.c_uint64), ("tier_edges", C.c_uint64)]


class DeviceView(C.Structure):
    _fields_ = [("values", C.c_void_p), ("row_end", C.c_void_p), ("src", C.c_void_p), ("stream", C.c_void_p),
                ("row_left", C.c_uint32), ("row_right", C.c_uint32), ("local_edges", C.c_uint64)]


def library_path():
    return _build.LIB


def declared_symbols():
    """Every function include/lux_b200.h declares (used by the no-GPU ABI test)."""
    text = open(_HEADER).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(luxb_[a-z0-9_]+)\s*\(", text)))


ABI_VERSION = 3  # must equal luxb_abi_version(): layout of luxb_config / luxb_stats_t / luxb_device_view


def load_library():
    """Load libluxb.so, building it in-tree if its sources are newer.  Raises (never falls back): a library that is
    missing, stale and not rebuildable, or built from another revision of the ABI is an error."""
    global _lib
    if _lib is not None:
        return _lib
    path = _build.LIB
    if _build.is_stale():
        try:
            _build.build()
        except Exception as e:  # noqa: BLE001
            raise LuxError("libluxb.so is %s and could not be built (%s); lux_b200 has no CPU fallback" % (
                "stale" if os.path.exists(path) else "missing", e))
    L = C.CDLL(path)
    L.luxb_last_error.restype = C.c_char_p
    L.luxb_version.restype = C.c_char_p
    L.luxb_close.restype = None
    if not hasattr(L, "luxb_abi_version") or L.luxb_abi_version() != ABI_VERSION:
        raise LuxError("libluxb.so at %s was built for another ABI revision than this binding (%d)" % (path, ABI_VERSION))
    _lib = L
    return L


def _chk(rc, what):
    if rc < 0:
        raise LuxError("%s failed (%d): %s" % (what, rc, load_library().luxb_last_error().decode()))
    return rc


def _p(a):
    return a.ctypes.data_as(C.c_void_p) if a is not None else None


def partition_csc(row_end, ne, P):
    """Reference partitioner on host arrays (pull_model.inl:108-131) -> (count, row_left, row_right, col_left)."""
    row_end = np.ascontiguousarray(row_end, np.uint64)
    rl, rr, cl = np.zeros(P, np.uint32), np.zeros(P, np.uint32), np.zeros(P, np.uint64)
    cnt = _chk(load_library().luxb_partition_csc(C.c_uint32(len(row_end)), C.c_uint64(ne), _p(row_end), C.c_int(P),
                                                 _p(rl), _p(rr), _p(cl)), "luxb_partition_csc")
    return cnt, rl, rr, cl


def write_lux(path, row_end, src, weight=None):
    """CSC arrays -> .lux file (tools/converter.cc layout); host only."""
    row_end = np.ascontiguousarray(row_end, np.uint64)
    src = np.ascontiguousarray(src, np.uint32)
    if weight is not None:
        weight = np.ascontiguousarray(weight, np.int32)
    csc = _Csc(len(row_end), len(src), _p(row_end), _p(src) if len(src) else None, _p(weight))
    _chk(load_library().luxb_write_lux(path.encode(), C.byref(csc)), "luxb_write_lux")


def convert_edgelist(edge_list_path, lux_path, nv, ne):
    """Text edge list ("src dst" per line) -> .lux, like tools/converter.cc -nv -ne -input -output; host only."""
    _chk(load_library().luxb_convert_edgelist(edge_list_path.encode(), lux_path.encode(), C.c_uint32(nv), C.c_uint64(ne)),
         "luxb_convert_edgelist")


_VDTYPE = {APP_PAGERANK: np.float32, APP_CC: np.uint32, APP_SSSP: np.uint32, APP_COLFILTER: np.float32,
           APP_SSSP_WEIGHTED: np.uint32, APP_BC: np.float64, APP_BC_WEIGHTED: np.float64,
           APP_TC: np.uint64, APP_KCORE: np.uint32, APP_TRUSS: np.uint32}


class LuxGraph:
    """One rank's handle.  Mirrors the phases of an app's top_level_task (pagerank/pagerank.cc:32-118):
    open (Graph::Graph + load) -> comm_init -> init -> iterate / run_to_convergence -> values / check."""

    def __init__(self, handle, app, rank, nranks):
        self._h = handle
        self.app, self.rank, self.nranks = app, rank, nranks
        nv, ne = C.c_uint32(), C.c_uint64()
        _chk(load_library().luxb_graph_info(self._h, C.byref(nv), C.byref(ne), None), "luxb_graph_info")
        self.nv, self.ne = nv.value, ne.value

    # ---- constructors -------------------------------------------------------------------------------------
    @staticmethod
    def _cfg(app, rank, nranks, device, start, exchange, verbose, zero_copy=False, balanced=False):
        return _Config(app, rank, nranks, device, start, exchange, 1 if verbose else 0, 1 if balanced else 0, 1 if zero_copy else 0)

    @classmethod
    def from_csc(cls, row_end, src, weight=None, app=APP_PAGERANK, rank=0, nranks=1, device=0, start=0,
                 exchange=EXCHANGE_NCCL, verbose=False, zero_copy=False, balanced=False):
        row_end = np.ascontiguousarray(row_end, np.uint64)
        src = np.ascontiguousarray(src, np.uint32)
        if weight is not None:
            weight = np.ascontiguousarray(weight, np.int32)
        csc = _Csc(len(row_end), len(src), _p(row_end), _p(src) if len(src) else None, _p(weight))
        cfg = cls._cfg(app, rank, nranks, device, start, exchange, verbose, zero_copy, balanced)
        h = C.c_void_p()
        _chk(load_library().luxb_open_csc(C.byref(csc), C.byref(cfg), C.byref(h)), "luxb_open_csc")
        return cls(h, app, rank, nranks)

    @classmethod
    def from_file(cls, path, app=APP_PAGERANK, rank=0, nranks=1, device=0, start=0, exchange=EXCHANGE_NCCL,
                  verbose=False):
        cfg = cls._cfg(app, rank, nranks, device, start, exchange, verbose)
        h = C.c_void_p()
        _chk(load_library().luxb_open_file(path.encode(), C.byref(cfg), C.byref(h)), "luxb_open_file")
        return cls(h, app, rank, nranks)

    @classmethod
    def from_rmat(cls, scale, nv, ne, seed, app=APP_PAGERANK, rank=0, nranks=1, device=0, start=0,
                  exchange=EXCHANGE_NCCL, verbose=False, zero_copy=False, balanced=False):
        cfg = cls._cfg(app, rank, nranks, device, start, exchange, verbose, zero_copy, balanced)
        h = C.c_void_p()
        _chk(load_library().luxb_open_rmat(C.c_int(scale), C.c_uint32(nv), C.c_uint64(ne), C.c_uint64(seed),
                                           C.byref(cfg), C.byref(h)), "luxb_open_rmat")
        return cls(h, app, rank, nranks)

    @classmethod
    def from_bipartite(cls, users, items, ratings, seed, rank=0, nranks=1, device=0, exchange=EXCHANGE_NCCL, balanced=False,
                       app=APP_COLFILTER, start=0):
        cfg = cls._cfg(app, rank, nranks, device, start, exchange, False, False, balanced)
        h = C.c_void_p()
        _chk(load_library().luxb_open_bipartite(C.c_uint32(users), C.c_uint32(items), C.c_uint64(ratings),
                                                C.c_uint64(seed), C.byref(cfg), C.byref(h)), "luxb_open_bipartite")
        return cls(h, app, rank, nranks)

    # ---- partition table ----------------------------------------------------------------------------------
    def bounds(self):
        P = self.nranks
        rl, rr, cl = np.zeros(P, np.uint32), np.zeros(P, np.uint32), np.zeros(P, np.uint64)
        fl, fr = np.zeros(P, np.uint64), np.zeros(P, np.uint64)
        found = _chk(load_library().luxb_partition_bounds(self._h, _p(rl), _p(rr), _p(cl), _p(fl), _p(fr)),
                     "luxb_partition_bounds")
        return dict(found=found, row_left=rl, row_right=rr, col_left=cl, fq_left=fl, fq_right=fr)

    def work_bounds(self):
        """The split the ranks work on (== bounds() unless opened with balanced=True)."""
        P = self.nranks
        rl, rr, cl = np.zeros(P, np.uint32), np.zeros(P, np.uint32), np.zeros(P, np.uint64)
        bal = _chk(load_library().luxb_work_bounds(self._h, _p(rl), _p(rr), _p(cl)), "luxb_work_bounds")
        return dict(balanced=bool(bal), row_left=rl, row_right=rr, col_left=cl)

    # ---- communicator -------------------------------------------------------------------------------------
    @staticmethod
    def comm_unique_id():
        buf = C.create_string_buffer(UNIQUE_ID_BYTES)
        _chk(load_library().luxb_comm_unique_id(buf), "luxb_comm_unique_id")
        return buf.raw

    def comm_init(self, unique_id):
        _chk(load_library().luxb_comm_init(self._h, unique_id), "luxb_comm_init")

    def comm_init_torch(self):
        """Ship the NCCL id over an already-initialised torch.distributed group (plumbing only)."""
        if self.nranks == 1:
            return
        import torch.distributed as dist
        obj = [self.comm_unique_id() if self.rank == 0 else None]
        dist.broadcast_object_list(obj, src=0)
        self.comm_init(obj[0])

    def p2p_connect_torch(self):
        """Exchange cudaIpc handles of the replicas so kernels / copy engines can write into peer HBM (exchange=P2P*).
        Collective and all-or-nothing: if the import fails on any rank, every rank falls back to the NCCL exchange.
        Returns True when the peer mappings are in place."""
        if self.nranks == 1:
            return True
        import torch
        import torch.distributed as dist
        L = load_library()
        ok = 1
        try:
            n = C.c_size_t(0)
            _chk(L.luxb_p2p_export(self._h, None, C.byref(n)), "luxb_p2p_export")
            buf = C.create_string_buffer(n.value)
            _chk(L.luxb_p2p_export(self._h, buf, C.byref(n)), "luxb_p2p_export")
            blob = buf.raw
        except LuxError:
            ok, blob, n = 0, b"", C.c_size_t(0)
        blobs = [None] * self.nranks
        dist.all_gather_object(blobs, blob)
        if ok and all(len(b) == n.value for b in blobs):
            if L.luxb_p2p_import(self._h, b"".join(blobs), C.c_size_t(n.value)) < 0:
                ok = 0
        else:
            ok = 0
        dev = "cuda" if dist.get_backend() == "nccl" else "cpu"
        flag = torch.tensor([ok], device=dev)
        dist.all_reduce(flag, op=dist.ReduceOp.MIN)
        if int(flag) == 0:
            L.luxb_p2p_disconnect(self._h)
            return False
        self._p2p = True
        return True

    # ---- phases -------------------------------------------------------------------------------------------
    def init(self):
        _chk(load_library().luxb_init(self._h), "luxb_init")
        return self

    def iterate(self, iters=1):
        active = C.c_uint64(0)
        _chk(load_library().luxb_iterate(self._h, C.c_int(iters), C.byref(active)), "luxb_iterate")
        return active.value

    def run_to_convergence(self, max_iters=0):
        it = C.c_int(0)
        _chk(load_library().luxb_run_to_convergence(self._h, C.c_int(max_iters), C.byref(it)),
             "luxb_run_to_convergence")
        return it.value

    def values(self, out=None):
        shape = (self.nv, CF_K) if self.app == APP_COLFILTER else (self.nv,)
        if out is None:
            out = np.empty(shape, _VDTYPE[self.app])
        _chk(load_library().luxb_get_values(self._h, _p(out), C.c_size_t(out.nbytes)), "luxb_get_values")
        return out

    def set_values(self, arr):
        arr = np.ascontiguousarray(arr, _VDTYPE[self.app])
        _chk(load_library().luxb_set_values(self._h, _p(arr), C.c_size_t(arr.nbytes)), "luxb_set_values")

    def local_range(self):
        v = self.device_view()
        return v.row_left, (v.row_right - v.row_left + 1) & 0xFFFFFFFF

    def local_values(self, out=None):
        """This rank's partition only (local order): D2H of (row_right - row_left + 1) values."""
        _, n = self.local_range()
        shape = (n, CF_K) if self.app == APP_COLFILTER else (n,)
        if out is None:
            out = np.empty(shape, _VDTYPE[self.app])
        _chk(load_library().luxb_get_local_values(self._h, _p(out), C.c_size_t(out.nbytes)), "luxb_get_local_values")
        return out

    def set_local_values(self, arr):
        """H2D of this rank's partition, then the device-side exchange (collective on nranks > 1)."""
        arr = np.ascontiguousarray(arr, _VDTYPE[self.app])
        _chk(load_library().luxb_set_local_values(self._h, _p(arr), C.c_size_t(arr.nbytes)), "luxb_set_local_values")

    def check(self):
        bad = C.c_uint64(0)
        _chk(load_library().luxb_check(self._h, C.byref(bad)), "luxb_check")
        return bad.value

    def stats(self):
        s = Stats()
        _chk(load_library().luxb_stats(self._h, C.byref(s)), "luxb_stats")
        return {k: getattr(s, k) for k, _ in Stats._fields_}

    def trace(self, max_entries=100000):
        a = np.zeros(max_entries, np.uint64)
        p = np.zeros(max_entries, np.int32)
        n = _chk(load_library().luxb_trace(self._h, _p(a), _p(p), C.c_int(max_entries)), "luxb_trace")
        return a[:n].copy(), p[:n].copy()

    def bc_run(self, sources):
        """Betweenness centrality (APP_BC handles, or APP_BC_WEIGHTED over weighted shortest paths, weights >= 1): add
        the dependencies of every source, in order, to the scores that values() returns.  Collective on nranks > 1 (every
        rank passes the same sources)."""
        s = np.ascontiguousarray(np.asarray(sources, dtype=np.int64).reshape(-1))
        if s.size and (s.min() < 0 or s.max() > 0xFFFFFFFF):
            raise LuxError("luxb_bc_run failed: source out of the u32 range")
        s = s.astype(np.uint32)
        _chk(load_library().luxb_bc_run(self._h, _p(s) if s.size else None, C.c_int(len(s))), "luxb_bc_run")

    def bc_source_state(self):
        """(lev u32 [nv], sigma f64 [nv], delta f64 [nv]) of the last source processed by bc_run; on an APP_BC_WEIGHTED
        handle lev is the weighted distance (INF = DIST_INF)."""
        lev = np.empty(self.nv, np.uint32)
        sigma = np.empty(self.nv, np.float64)
        delta = np.empty(self.nv, np.float64)
        _chk(load_library().luxb_bc_source_state(self._h, _p(lev), _p(sigma), _p(delta), C.c_size_t(self.nv)),
             "luxb_bc_source_state")
        return lev, sigma, delta

    def tc_run(self):
        """Triangle counting (APP_TC handles): recount the triangles at every vertex of the undirected simple graph (the
        u64 values() returns) and return the total.  Collective on nranks > 1."""
        total = C.c_uint64(0)
        _chk(load_library().luxb_tc_run(self._h, C.byref(total)), "luxb_tc_run")
        return total.value

    def kcore_run(self):
        """k-core decomposition (APP_KCORE handles): recompute the core number of every vertex of the undirected simple
        graph (the u32 values() returns) and return the degeneracy (the largest core number).  Collective on
        nranks > 1."""
        degeneracy = C.c_uint32(0)
        _chk(load_library().luxb_kcore_run(self._h, C.byref(degeneracy)), "luxb_kcore_run")
        return degeneracy.value

    def truss_run(self):
        """k-truss decomposition (APP_TRUSS handles): recompute the support and truss number of every edge of the
        undirected simple graph (values() returns the vertex truss, the largest truss number at each vertex) and return
        kmax.  Collective on nranks > 1."""
        kmax = C.c_uint32(0)
        _chk(load_library().luxb_truss_run(self._h, C.byref(kmax)), "luxb_truss_run")
        return kmax.value

    def truss_num_edges(self):
        m = C.c_uint64(0)
        _chk(load_library().luxb_truss_num_edges(self._h, C.byref(m)), "luxb_truss_num_edges")
        return m.value

    def truss_edges(self):
        """(lo, hi, support, truss), u32 [m] each, edges in ascending (lo, hi) order with lo < hi; support of the input
        graph, truss numbers of the last run (zeros before the first)."""
        m = self.truss_num_edges()
        lo, hi, sup, tr = (np.empty(m, np.uint32) for _ in range(4))
        _chk(load_library().luxb_truss_edges(self._h, _p(lo), _p(hi), _p(sup), _p(tr), C.c_uint64(m)), "luxb_truss_edges")
        return lo, hi, sup, tr

    def set_truss(self, truss):
        """Overwrite the truss numbers (u32 [m], the order of truss_edges()) so that check() judges them."""
        t = np.ascontiguousarray(truss, np.uint32)
        _chk(load_library().luxb_truss_set_truss(self._h, _p(t) if t.size else None, C.c_uint64(t.size)), "luxb_truss_set_truss")

    def enable_kernel_timing(self, on=True):
        _chk(load_library().luxb_enable_kernel_timing(self._h, C.c_int(1 if on else 0)), "luxb_enable_kernel_timing")

    def out_degree(self, out=None):
        if out is None:
            out = np.empty(self.nv, np.uint32)
        _chk(load_library().luxb_get_out_degree(self._h, _p(out), C.c_size_t(out.nbytes)), "luxb_get_out_degree")
        return out

    def debug_gather_ms(self, packed=True):
        ms = C.c_float(0)
        _chk(load_library().luxb_debug_gather_ms(self._h, C.c_int(1 if packed else 0), C.byref(ms)), "luxb_debug_gather_ms")
        return ms.value

    def device_view(self):
        v = DeviceView()
        _chk(load_library().luxb_device_view_get(self._h, C.byref(v)), "luxb_device_view_get")
        return v

    def local_csc(self, weighted=False):
        v = self.device_view()
        n = (v.row_right - v.row_left + 1) & 0xFFFFFFFF
        re_ = np.empty(n, np.uint64)
        src = np.empty(v.local_edges, np.uint32)
        w = np.empty(v.local_edges, np.int32) if weighted else None
        _chk(load_library().luxb_get_local_csc(self._h, _p(re_), _p(src), _p(w)), "luxb_get_local_csc")
        return (re_, src, w) if weighted else (re_, src)

    def close(self):
        if self._h:
            if getattr(self, "_p2p", False):
                # exported buffers may only be freed once every importer has unmapped them
                load_library().luxb_p2p_disconnect(self._h)
                try:
                    import torch.distributed as dist
                    if dist.is_initialized():
                        dist.barrier()
                except Exception:  # noqa: BLE001
                    pass
                self._p2p = False
            load_library().luxb_close(self._h)
            self._h = None

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()
