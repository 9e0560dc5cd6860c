"""lux_b200 — H100-native replacement for the hot path of LuxGraph/Lux.

Host side: a thin ctypes mirror of include/lux_b200.h.  All compute is in lux_b200/_lib/libluxb.so (hand-written
sm_90a CUDA).  There is NO CPU fallback: importing works anywhere (so the ABI can be inspected), but opening a
graph without the library or without a GPU raises.
"""
from .binding import (APP_PAGERANK, APP_CC, APP_SSSP, APP_COLFILTER, APP_SSSP_WEIGHTED, APP_BC, APP_BC_WEIGHTED, APP_TC, APP_KCORE, APP_TRUSS, DIST_INF,
                      EXCHANGE_NCCL, EXCHANGE_P2P, EXCHANGE_P2P_FUSED, DENSE_BITMAP, SPARSE_QUEUE, CF_K, LuxError, LuxGraph,
                      load_library, partition_csc, library_path, declared_symbols, write_lux, convert_edgelist)
from .apps import pagerank, components, sssp, colfilter, betweenness, triangles, core_number, truss  # noqa: F401

__all__ = ["APP_PAGERANK", "APP_CC", "APP_SSSP", "APP_COLFILTER", "APP_SSSP_WEIGHTED", "APP_BC", "APP_BC_WEIGHTED", "APP_TC", "APP_KCORE", "APP_TRUSS", "DIST_INF",
           "EXCHANGE_NCCL", "EXCHANGE_P2P", "EXCHANGE_P2P_FUSED", "DENSE_BITMAP", "SPARSE_QUEUE", "CF_K", "LuxError", "LuxGraph",
           "load_library", "partition_csc", "library_path", "declared_symbols", "write_lux", "convert_edgelist", "pagerank",
           "components", "sssp", "colfilter", "betweenness", "triangles", "core_number", "truss"]
