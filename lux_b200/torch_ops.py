"""PyTorch front-end of the C ABI (SURVEY §8 f4): the four Lux apps, weighted SSSP, betweenness centrality, triangle counting, k-core decomposition and k-truss decomposition as `torch.ops.luxb.*` custom ops taking the CSC as
torch tensors and returning torch tensors.  Plumbing only — every op opens a libluxb handle through the ctypes binding
(lux_b200/binding.py), runs the app on the CUDA device of the current torch context and copies the result back; no torch
kernel takes part in the computation, and there is no CPU fallback (the ops raise without a GPU).

    import lux_b200.torch_ops            # registers the ops
    ranks  = torch.ops.luxb.pagerank(row_end, src, 10)          # f32 [nv]  (rank / out-degree, pagerank_gpu.cu:98-100)
    labels = torch.ops.luxb.components(row_end, src)            # i64 [nv]  (max reaching id, components_gpu.cu:112-122)
    dist   = torch.ops.luxb.sssp(row_end, src, 0)               # i64 [nv]  (hop count, INF = nv, sssp_gpu.cu:122)
    x      = torch.ops.luxb.colfilter(row_end, src, weight, 10) # f32 [nv, 20]
    dist   = torch.ops.luxb.sssp_weighted(row_end, src, weight, 0)  # i64 [nv]  (weighted distance, INF = 2^32 - 1)
    bc     = torch.ops.luxb.betweenness(row_end, src, sources)  # f64 [nv]  (Σ over sources of Brandes' δ, not normalised)
    bc     = torch.ops.luxb.betweenness_weighted(row_end, src, weight, sources)  # f64 [nv]  (weighted paths, weights >= 1)
    t      = torch.ops.luxb.triangles(row_end, src)             # i64 [nv]  (triangles at each vertex, undirected simple graph)
    core   = torch.ops.luxb.core_number(row_end, src)           # i64 [nv]  (core number of each vertex, undirected simple graph)
    edges, truss = torch.ops.luxb.k_truss(row_end, src)         # i64 [m, 2] (lo, hi ascending), i64 [m] truss numbers
row_end: int64 [nv] END offsets (the .lux convention); src: int64/int32 [ne]; weight: int32 [ne]; sources: int64/int32 [k] vertex ids."""
import numpy as np
import torch

from . import apps as _apps


def _np(t, dtype):
    return np.ascontiguousarray(t.detach().cpu().numpy()).astype(dtype, copy=False)


def _device_index(t):
    return t.device.index if t.is_cuda and t.device.index is not None else (torch.cuda.current_device() if torch.cuda.is_available() else 0)


_lib = torch.library.Library("luxb", "DEF")
_lib.define("pagerank(Tensor row_end, Tensor src, int num_iter) -> Tensor")
_lib.define("components(Tensor row_end, Tensor src) -> Tensor")
_lib.define("sssp(Tensor row_end, Tensor src, int start) -> Tensor")
_lib.define("colfilter(Tensor row_end, Tensor src, Tensor weight, int num_iter) -> Tensor")
_lib.define("sssp_weighted(Tensor row_end, Tensor src, Tensor weight, int start) -> Tensor")
_lib.define("betweenness(Tensor row_end, Tensor src, Tensor sources) -> Tensor")
_lib.define("betweenness_weighted(Tensor row_end, Tensor src, Tensor weight, Tensor sources) -> Tensor")
_lib.define("triangles(Tensor row_end, Tensor src) -> Tensor")
_lib.define("core_number(Tensor row_end, Tensor src) -> Tensor")
_lib.define("k_truss(Tensor row_end, Tensor src) -> (Tensor, Tensor)")


def _pagerank(row_end, src, num_iter):
    out = _apps.pagerank(_np(row_end, np.uint64), _np(src, np.uint32), num_iter=int(num_iter), device=_device_index(row_end))
    return torch.from_numpy(out).to(row_end.device)


def _components(row_end, src):
    out = _apps.components(_np(row_end, np.uint64), _np(src, np.uint32), device=_device_index(row_end))
    return torch.from_numpy(out["labels"].astype(np.int64)).to(row_end.device)


def _sssp(row_end, src, start):
    out = _apps.sssp(_np(row_end, np.uint64), _np(src, np.uint32), start=int(start), device=_device_index(row_end))
    return torch.from_numpy(out["labels"].astype(np.int64)).to(row_end.device)


def _colfilter(row_end, src, weight, num_iter):
    out = _apps.colfilter(_np(row_end, np.uint64), _np(src, np.uint32), _np(weight, np.int32), num_iter=int(num_iter),
                          device=_device_index(row_end))
    return torch.from_numpy(out).to(row_end.device)


def _sssp_weighted(row_end, src, weight, start):
    out = _apps.sssp(_np(row_end, np.uint64), _np(src, np.uint32), start=int(start), device=_device_index(row_end),
                     weight=_np(weight, np.int32))
    return torch.from_numpy(out["labels"].astype(np.int64)).to(row_end.device)


def _betweenness(row_end, src, sources):
    out = _apps.betweenness(_np(row_end, np.uint64), _np(src, np.uint32), sources=_np(sources, np.int64), device=_device_index(row_end))
    return torch.from_numpy(out).to(row_end.device)


def _betweenness_weighted(row_end, src, weight, sources):
    out = _apps.betweenness(_np(row_end, np.uint64), _np(src, np.uint32), sources=_np(sources, np.int64), device=_device_index(row_end),
                            weight=_np(weight, np.int32))
    return torch.from_numpy(out).to(row_end.device)


def _triangles(row_end, src):
    out = _apps.triangles(_np(row_end, np.uint64), _np(src, np.uint32), device=_device_index(row_end))
    return torch.from_numpy(out["per_vertex"].astype(np.int64)).to(row_end.device)


def _core_number(row_end, src):
    out = _apps.core_number(_np(row_end, np.uint64), _np(src, np.uint32), device=_device_index(row_end))
    return torch.from_numpy(out["core"].astype(np.int64)).to(row_end.device)


def _k_truss(row_end, src):
    out = _apps.truss(_np(row_end, np.uint64), _np(src, np.uint32), device=_device_index(row_end))
    edges = np.stack([out["lo"], out["hi"]], axis=1).astype(np.int64).reshape(-1, 2)
    return torch.from_numpy(edges).to(row_end.device), torch.from_numpy(out["truss"].astype(np.int64)).to(row_end.device)


for _name, _fn in (("pagerank", _pagerank), ("components", _components), ("sssp", _sssp), ("colfilter", _colfilter),
                   ("sssp_weighted", _sssp_weighted), ("betweenness", _betweenness), ("betweenness_weighted", _betweenness_weighted),
                   ("triangles", _triangles), ("core_number", _core_number), ("k_truss", _k_truss)):
    _lib.impl(_name, _fn, "CompositeExplicitAutograd")
