"""Inputs on which the pull sweeps' fp32 units sum exactly while vertex sums outgrow fp32 (tests/test_gpu_wide_exact.py,
tests/test_wide_exact_model.py), and the configuration facts they are sized by: the hotness order and tier-0 slots."""
import numpy as np

import oracle as O
from graphs import in_degrees, mix32


FP32_EXACT = (1 << 24) - 1  # the largest integer below which every integer is a float32
WIDE_MIN = 1 << 25           # a vertex sum at or above this is "wide": fp32 keeps only every fourth integer there


def hot_order(row_end, src, hot_mb=24.0, cap=4096):
    """The hot set of build_hot_layout (lux_b200/csrc/api.cu) in hotness order (hot_select_kernel, build.cuh): the
    vertices of out-degree >= tau, tau >= 2 the smallest threshold whose set fits in hot_mb MB of values (degrees
    clamped at `cap` for the threshold only), ordered by descending out-degree, ties by ascending id.  The panel cuts
    this order into blocks of LUXB_SB_BS values; tier 0 is its first min(H, LUXB_SB_BLOCKS * BS) entries."""
    nv = len(row_end)
    deg = O.out_degree(nv, src)
    h_max = min(int(hot_mb * 1e6 / 4.0), nv)
    if h_max == 0 or nv < 2:
        return np.zeros(0, np.int64)
    hist = np.bincount(np.minimum(deg, cap), minlength=cap + 1)
    above, tau = 0, cap + 1
    for d in range(cap, 1, -1):
        if above + int(hist[d]) > h_max:
            break
        above += int(hist[d])
        tau = d
    ids = np.nonzero(deg >= tau)[0]
    return ids[np.lexsort((ids, -deg[ids].astype(np.int64)))]


def max_multiplicity(row_end, src):
    """The largest number of parallel edges between one (source, destination) pair."""
    if len(src) == 0:
        return 0
    dst = np.repeat(np.arange(len(row_end), dtype=np.uint64), in_degrees(row_end))
    _, cnt = np.unique((dst << np.uint64(32)) | src.astype(np.uint64), return_counts=True)
    return int(cnt.max())


def tier0_panel(row_end, src, bs, blocks, min_indeg, hot_mb=24.0):
    """The tier-0 panel of the source-blocked split: (block of every source, -1 outside tier 0; the most edges of one
    (block, hub) slot).  Tier 0 is the first min(H, blocks * bs) vertices of the hotness order, cut into blocks of bs;
    every edge from one of them into a hub (in-degree >= min_indeg) goes to its block's slot for that hub.  A slot has
    at most bs * max_multiplicity edges; the count here is the one the graph reaches."""
    nv = len(row_end)
    order = hot_order(row_end, src, hot_mb)
    n0 = min(len(order), blocks * bs)
    blk = np.full(nv, -1, np.int64)
    blk[order[:n0]] = np.arange(n0) // bs
    indeg = in_degrees(row_end)
    dst = np.repeat(np.arange(nv), indeg)
    sel = (indeg[dst] >= min_indeg) & (blk[src] >= 0)
    slot = dst[sel].astype(np.int64) * blocks + blk[src[sel]]
    most = int(np.unique(slot, return_counts=True)[1].max()) if slot.size else 0
    assert most <= bs * max_multiplicity(row_end, src)
    return blk, most


def vertex_sums(row_end, src, x):
    """S[v] = sum of x over v's in-edges, exact in fp64 for integer x (sums below 2^53)."""
    dst = np.repeat(np.arange(len(row_end)), in_degrees(row_end))
    return np.bincount(dst, weights=x[src].astype(np.float64), minlength=len(row_end))


def wide_vertices(s):
    """Vertices whose sum is wide and not a float32: there a single fp32 rounding of S, and any extra rounding of a
    partial sum above 2^24, are visible in the stored value."""
    return (s >= WIDE_MIN) & (s != s.astype(np.float32).astype(np.float64))


def wide_exact_pr_inputs(nv, unit_edges, wide=None, salt=0):
    """PageRank values whose vertex sums S outgrow fp32 while every fp32 unit of the sweep stays exact.

    The sweeps sum edges in fp32 only inside units of at most `unit_edges` edges (a warp round or piece of the flagged
    stream, a merge-path tile, a panel slot, a hub's main part) and combine units in fp64, narrowing once.  Sources where
    `wide` is set (all by default) get integers in {1..K}, K = floor((2^24 - 1) / unit_edges), the others 1; so a unit
    that only sees `wide` sources in at most unit_edges edges, or at most 2^24 - 1 edges of the others, sums exactly.
    The device must then return update(rn32(S)), which is what the oracle computes, while S itself reaches 2^25 and
    beyond: an fp64 carry or combine narrowed to fp32 rounds S more than once and moves the result."""
    k = FP32_EXACT // max(int(unit_edges), 1)
    assert k >= 2, "unit of %d edges: no room for values above 1" % unit_edges
    x = (np.uint64(1) + mix32(np.arange(nv, dtype=np.uint64), salt + 17) % np.uint64(k)).astype(np.float32)
    if wide is not None:
        x[~np.asarray(wide, bool)] = 1.0
    return x


def wide_exact_cf_inputs(users, items):
    """exact_cf_inputs with the items' integers raised from {1..b}, b <= 8, to {1..b}, b = floor((2^24 - 1) / (40 * 256)):
    one 256-edge chunk of cf_chunk_kernel then sums at most 256 terms |err * x_u| <= 2 * 20 b of one sign exactly in
    fp32, and cf_update_kernel adds the chunk partials in fp64 without rounding.  An item's accumulator reaches far past
    2^24, so factors 10-19 = rn(GAMMA * rn32(acc)) see any fp32 step in the combination of the chunks."""
    b = FP32_EXACT // (40 * 256)
    x = np.zeros((users + items, 20), np.float32)
    uid = np.arange(users, dtype=np.uint64)
    x[:users] = (np.uint64(1) + ((mix32(uid, 1)[:, None] >> np.arange(20, dtype=np.uint64)) & np.uint64(1))).astype(np.float32)
    iid = np.arange(items, dtype=np.uint64)
    h = mix32(iid, 2)[:, None] ^ mix32(np.arange(10, dtype=np.uint64), 3)[None, :]
    x[users:, :10] = (np.uint64(1) + h % np.uint64(b)).astype(np.float32)
    return x


def regular_indegree(n, d, seed=3):
    """n vertices, each with exactly d in-edges from random sources (sorted per vertex): with d a multiple of a flagged
    stream's piece length, every vertex's in-edges fill whole pieces, and no vertex starts or ends inside a piece."""
    rng = np.random.default_rng(seed)
    s = np.sort(rng.integers(0, n, (n, d)), axis=1).reshape(-1)
    return O.edges_to_csc(n, s, np.repeat(np.arange(n), d))
