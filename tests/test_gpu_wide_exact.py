"""Exact-arithmetic parity of the pull sweeps and collaborative filtering on inputs whose sums outgrow fp32: the fp64
carries and combines of every sweep path, pinned bit for bit.

The inputs of tests/test_gpu_exact.py keep every vertex sum below 2^21, where fp32 is exact in any order: they pin the
routing of every edge but would pass unchanged if an fp64 step of the sweeps had been narrowed to fp32.  Here the values
come from wide_inputs.wide_exact_pr_inputs / wide_exact_cf_inputs: every fp32 unit of the path under test (a warp round or
piece of the flagged stream, a merge-path tile, a panel slot, a hub's main part, a 256-edge CF chunk) sums exactly,
while many vertex sums pass 2^25 and are not floats.  The device must then return update(rn32(S)), which is the
oracle's result, and any extra fp32 rounding of a partial sum above 2^24 moves it.  Each case is one set_values +
iterate(1) against one oracle iteration, compared by the bits, and first asserts that its inputs are not vacuous:
a per-case least number of vertices with S >= 2^25 and S != rn32(S).  tests/test_wide_exact_model.py proves on the
CPU that a model of the units matches the oracle on these inputs and that each narrowed step does not.

Covered: the plain flagged stream in all 8 main shapes (a 2^20-leaf star, RMAT-17, and one vertex per 1024-edge piece for
the round-to-round carry), both fix-ups at RMAT-22 over several rounds on one handle, the merge path in every pull shape
with and without zero-copy edges, the forced split's tier 0 in all 6 panel shapes and with the concurrent panel
schedule on 1, 8 and the default number of SMs, the forced cold-hub stream, PageRank at 2, 3 and 4 emulated ranks
(plain and balanced split), CF at the hub-item size and at C5, and a crafted CF graph around the chunk and group
edges.  The fused fix-up's run-dependent fp64 association is bounded on ordinary values at RMAT-22.
LUXB_SKIP_HEAVY=1 skips C5."""
import functools
import os

import numpy as np
import pytest

import oracle as O
import lux_b200 as L
from emu_ranks import emulate, run_ranks
from graphs import rmat
from wide_inputs import (WIDE_MIN, hot_order, regular_indegree, tier0_panel, vertex_sums, wide_exact_cf_inputs,
                         wide_exact_pr_inputs, wide_vertices)
from test_gpu_exact import CF_GAMMA, assert_bit_equal, set_env

pytestmark = pytest.mark.gpu
heavy = pytest.mark.skipif(os.environ.get("LUXB_SKIP_HEAVY") == "1", reason="LUXB_SKIP_HEAVY=1")

# edges per piece of the main flagged-stream shapes (LUXB_SEG_MAIN_SHAPES in api.cu: rounds x 256) and per merge-path
# tile (LUXB_PULL_SHAPES: 32 lanes x items per lane; a tile's edges are at most its items)
MAIN_PIECE = [512, 256, 256, 1024, 256, 256, 256, 512]
MERGE_TILE = [7 * 32, 9 * 32, 7 * 32]
ROUND = 256


@functools.lru_cache(maxsize=None)
def graph(name):
    if name == "star_2^20":  # vertex 0 with 2^20 in-edges, from 1 .. 2^20
        n = 1 << 20
        return O.edges_to_csc(n + 1, np.arange(1, n + 1), np.zeros(n, np.int64))
    if name == "one_vertex_per_piece":
        return regular_indegree(2048, 1024)
    if name == "uniform_256":  # every vertex a hub; a tier-0 slot holds a few edges, a hub adds 48 of them
        return regular_indegree(32768, 256)
    return rmat(int(name[len("rmat"):]))


def wide_step(g, row_end, src, x, min_wide, what):
    """One set_values + iterate(1) from x, bit for bit against the oracle, after asserting x is not vacuous."""
    n_wide = int(wide_vertices(vertex_sums(row_end, src, x)).sum())
    assert n_wide >= min_wide, "%s: %d wide vertices, want >= %d" % (what, n_wide, min_wide)
    g.set_values(x)
    g.iterate(1)
    assert_bit_equal(g.values(), O.pagerank_iter(row_end, src, O.out_degree(len(row_end), src), x), what)


def run_wide(name, unit, min_wide, rounds=1, wide=None, **kw):
    row_end, src = graph(name)
    with L.LuxGraph.from_csc(row_end, src, **kw) as g:
        g.init()
        st = g.stats()
        for r in range(rounds):
            wide_step(g, row_end, src, wide_exact_pr_inputs(len(row_end), unit, wide, salt=r), min_wide,
                      "%s round %d" % (name, r))
    return st


# ---- 1. the plain flagged stream ---------------------------------------------------------------------------------------
@pytest.mark.parametrize("main_shape", range(8))
def test_plain_stream_every_main_shape(main_shape, monkeypatch):
    """Units: the shape's piece (head / tail partials) and round.  The star's one hub spans thousands of pieces; RMAT-17
    has 10 wide vertices at the 1024-edge pieces' K = 16383 and more at shorter pieces (at least 8 asserted)."""
    set_env(monkeypatch, dict(LUXB_SB=0, LUXB_SEG_MAIN_SHAPE=main_shape))
    for name, min_wide in (("star_2^20", 1), ("rmat17", 8)):
        assert run_wide(name, MAIN_PIECE[main_shape], min_wide)["panel_edges"] == 0


def test_plain_stream_round_carry(monkeypatch):
    """Main shape 3 (pieces of four 256-edge rounds) on 2048 vertices of in-degree 1024: each vertex is one piece, its
    sum the fp64 carry across four rounds, narrowed once, so the unit is the round (K = 65535).  Mean S = 2^25: at
    least 500 wide vertices.  The only main shape with more than two rounds per piece, where a narrowed carry shows."""
    set_env(monkeypatch, dict(LUXB_SB=0, LUXB_SEG_MAIN_SHAPE=3))
    run_wide("one_vertex_per_piece", ROUND, 500)


# ---- 2. both fix-ups at RMAT-22 -----------------------------------------------------------------------------------------
@functools.lru_cache(maxsize=1)
def rmat22():
    return O.gen_rmat_csc(22, 1 << 22, 16 << 22, 27)


@pytest.mark.parametrize("fused", [0, 1])
def test_fixups_rmat22_several_rounds(fused, monkeypatch):
    """Main shape 6 (256-edge pieces, 1025 fix-up blocks), K = 65535: a sum passes 2^25 from about 1024 in-edges on, and
    RMAT-22 has thousands of such vertices (at least 1000 asserted).  Three rounds on one handle."""
    set_env(monkeypatch, dict(LUXB_FUSED_FIXUP=fused, LUXB_SB=0, LUXB_SEG_MAIN_SHAPE=6))
    row_end, src = rmat22()
    with L.LuxGraph.from_rmat(22, 1 << 22, 16 << 22, 27) as g:
        g.init()
        assert g.stats()["panel_edges"] == 0
        for r in range(3):
            wide_step(g, row_end, src, wide_exact_pr_inputs(len(row_end), 256, salt=r), 1000, "rmat22 fused=%d round %d" % (fused, r))


def ulp_distance(a, b):
    """|a - b| in float32 ulps, for finite values of one sign."""
    return np.abs(a.view(np.int32).astype(np.int64) - b.view(np.int32).astype(np.int64))


def test_fused_fixup_association_bound(monkeypatch, capsys):
    """The fused fix-up combines tail partials in tile order, but its fp64 association depends on which block prefixes
    were published when a block looked back; the three-kernel fix-up's association is fixed.  On ordinary values two
    fp64 sums of the same <= 2^18 fp32 partials differ by far less than an fp32 ulp of S (relative 2^18 * 2^-53), so
    rn32 of them differs by at most one ulp, and only when they straddle a rounding boundary.  One ulp of acc moves
    fma(0.15, acc, init) by at most one ulp of y after its rounding, and the division by the out-degree rounds that once
    more: at most two ulps in the stored value.  Asserted on every vertex; on wide exact inputs the two agree bit for
    bit."""
    row_end, src = rmat22()
    deg = O.out_degree(len(row_end), src)
    x = O.pagerank_iter(row_end, src, deg, O.pagerank_init(deg))  # ordinary values: one step from the initial ranks
    xw = wide_exact_pr_inputs(len(row_end), 256)
    out = {}
    for fused in (0, 1):
        set_env(monkeypatch, dict(LUXB_FUSED_FIXUP=fused, LUXB_SB=0, LUXB_SEG_MAIN_SHAPE=6))  # 1025 fix-up blocks
        with L.LuxGraph.from_rmat(22, 1 << 22, 16 << 22, 27) as g:
            g.init()
            g.set_values(x)
            g.iterate(1)
            a = g.values()
            g.set_values(xw)
            g.iterate(1)
            out[fused] = (a, g.values())
    d = ulp_distance(out[0][0], out[1][0])
    with capsys.disabled():
        print("\nfused vs three-kernel fix-up, RMAT-22, ordinary values: %d of %d vertices differ, at most %d ulp" % (
            int((d > 0).sum()), len(d), int(d.max())))
    assert int(d.max()) <= 2
    assert_bit_equal(out[1][1], out[0][1], "fused vs three-kernel, wide exact inputs")


# ---- 3. the merge path -------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("zero_copy", [False, True])
@pytest.mark.parametrize("pull_shape", [0, 1, 2])
def test_merge_path_every_pull_shape(pull_shape, zero_copy, monkeypatch):
    """Unit: the tile (224 or 288 edges, K = 74897 or 58253).  RMAT-17 has over 100 wide vertices there."""
    env = dict(LUXB_PULL_SHAPE=pull_shape)
    if not zero_copy:
        env["LUXB_SWEEP"] = "merge"
    set_env(monkeypatch, env)
    for name, min_wide in (("star_2^20", 1), ("rmat17", 100)):
        assert run_wide(name, MERGE_TILE[pull_shape], min_wide, zero_copy=zero_copy)["panel_edges"] == 0


# ---- 4. the forced split: tier 0, the concurrent panel schedule, the cold-hub stream -----------------------------------
BS, BLOCKS, MIN_INDEG = 512, 48, 16


def run_panel(env, monkeypatch, min_wide, hot_mb=24.0, cold=False):
    """uniform_256 with tier-0 sources at values up to K = (2^24 - 1) / (most edges of one slot), the rest 1: slots, the
    hubs' main parts and the cold slots (cold sources: 1) all sum exactly.  The configuration is the one the rule of
    wide_inputs.hot_order implies: H hot vertices, min(H, 48 * 512) of them in tier 0, every vertex a hub."""
    set_env(monkeypatch, dict(env, LUXB_SB=1, LUXB_SB_BS=BS, LUXB_SB_BLOCKS=BLOCKS, LUXB_SB_MIN_INDEG=MIN_INDEG,
                              LUXB_HOT_MB=hot_mb, LUXB_CS=1 if cold else 0))
    row_end, src = graph("uniform_256")
    blk, most = tier0_panel(row_end, src, BS, BLOCKS, MIN_INDEG, hot_mb)
    st = run_wide("uniform_256", max(most, MIN_INDEG), min_wide, wide=blk >= 0)
    hot = len(hot_order(row_end, src, hot_mb))
    assert st["panel_blocks"] == -(-min(hot, BLOCKS * BS) // BS) and st["panel_hubs"] == len(row_end), st
    assert (st["cold_hub_edges"] > 0) == cold, st
    return st


@pytest.mark.parametrize("panel_shape", range(6))
def test_panel_tier0_every_panel_shape(panel_shape, monkeypatch):
    """48 blocks of 512 tier-0 sources, slots of at most about 20 edges: most hubs are wide (10 000 asserted)."""
    run_panel(dict(LUXB_SEG_PANEL_SHAPE=panel_shape, LUXB_SEG_MAIN_SHAPE=(panel_shape + 2) % 8), monkeypatch, 10000)


@pytest.mark.parametrize("panel_sms", [1, 8, None])
def test_panel_concurrent_schedule(panel_sms, monkeypatch):
    """The panel sweep beside the L1-gather sweeps on LUXB_PANEL_SMS SMs (None: the default)."""
    run_panel({} if panel_sms is None else dict(LUXB_PANEL_SMS=panel_sms), monkeypatch, 10000)


def test_cold_hub_stream(monkeypatch):
    """A hot set of 10 000 values: the rest of the sources are cold, and their hub edges go to the cold-hub stream
    (values 1, at most a hub's in-degree per slot).  A hub's tier-0 part is then about a third of its in-edges: at
    least 1000 wide hubs."""
    run_panel(dict(LUXB_CS_SEG_MB=0.02), monkeypatch, 1000, hot_mb=0.04, cold=True)


# ---- 5. PageRank on emulated ranks ---------------------------------------------------------------------------------------
def case_pagerank_wide(world, balanced):
    """1024 vertices of in-degree 8192: every destination range cuts no vertex's in-edges, each vertex's sum passes 2^25
    at the 1024-edge pieces' K (887 of 1024 are wide; at least 800 asserted), and every rank must match the oracle."""
    row_end, src = regular_indegree(1024, 8192)
    x = wide_exact_pr_inputs(len(row_end), 1024)

    def body(rank, uid):
        with L.LuxGraph.from_csc(row_end, src, rank=rank, nranks=world, device=0, balanced=balanced) as g:
            g.comm_init(uid(0))
            g.init()
            wide_step(g, row_end, src, x, 800, "rank %d of %d balanced=%s" % (rank, world, balanced))

    run_ranks(world, body)


@pytest.mark.parametrize("balanced", [False, True])
def test_pagerank_emulated_ranks(balanced, monkeypatch):
    rc, out = emulate("test_gpu_wide_exact", "case_pagerank_wide", env=None if balanced else dict(LUXB_SB=0),
                      worlds=[2, 3, 4], balanced=balanced)
    assert rc == 0, out[-6000:]


# ---- 6. collaborative filtering ------------------------------------------------------------------------------------------
def cf_wide_step(g, row_end, src, w, users, what, min_wide_share=None, min_wide=None):
    """Items' factors 10-19 = rn(GAMMA * rn32(acc)) bit for bit; every other value within 2e-6 of the magnitude of the
    terms of x + GAMMA * (acc - LAMBDA * x) (FMA contraction of that update moves it by an ulp of its largest term,
    which for a wide acc and an item value near GAMMA * |acc| is far more than 2e-6 of the small result)."""
    items = len(row_end) - users
    x = wide_exact_cf_inputs(users, items)
    g.set_values(x)
    g.iterate(1)
    gpu = g.values()
    ref = O.cf_iter(row_end, src, w, x)
    # |acc| from the exact factors: rn(GAMMA * rn32(acc)) / GAMMA is within 2^-22 relative of acc
    acc = np.abs(ref[users:, 10:].astype(np.float64)) / float(CF_GAMMA)
    n_wide = int((acc >= WIDE_MIN * (1 + 2 ** -20)).sum())
    want = min_wide if min_wide is not None else int(min_wide_share * acc.size)
    assert n_wide >= want, "%s: %d wide accumulators, want >= %d" % (what, n_wide, want)
    assert_bit_equal(gpu[users:, 10:].reshape(-1), ref[users:, 10:].reshape(-1), what + ", items' factors 10-19")
    scale = np.abs(x).astype(np.float64) + np.abs(ref.astype(np.float64) - x)
    bad = np.abs(gpu.astype(np.float64) - ref) > 2e-6 * scale
    assert not bad.any(), "%s: %d values off by more than 2e-6 of their terms" % (what, int(bad.sum()))


def test_colfilter_hub_items():
    """20 000 users, 300 items, 1.5 M ratings: about 60 % of the accumulators pass 2^25 (half asserted)."""
    users, items, ratings = 20000, 300, 1500000
    with L.LuxGraph.from_bipartite(users, items, ratings, 5) as g:
        row_end, src, w = g.local_csc(weighted=True)
        g.init()
        cf_wide_step(g, row_end, src, w, users, "hub items", min_wide_share=0.5)


@heavy
def test_colfilter_c5():
    """C5: 480 189 users, 17 770 items, 100 M ratings; at least a quarter of the accumulators pass 2^25."""
    users, items, ratings = 480189, 17770, 100480507
    with L.LuxGraph.from_bipartite(users, items, ratings, 5) as g:
        row_end, src, w = g.local_csc(weighted=True)
        g.init()
        cf_wide_step(g, row_end, src, w, users, "C5", min_wide_share=0.25)


CRAFTED_INDEG = [0, 1, 15, 16, 17, 255, 256, 257, 511, 512, 513, 4097]


def test_colfilter_crafted_chunk_edges():
    """Items of in-degree 0, 1, 15-17 (the 16-edge group stride of cf_chunk_kernel), 255-257 and 511-513 (one and two
    256-edge chunks) and 4097 (17 chunks, wide); 3000 users without in-edges (their update is from acc = 0).  Every
    item and user is held to the oracle; at least the 4097-edge item is wide on all ten exact factors."""
    users = 3000
    rng = np.random.default_rng(8)
    s = [np.sort(rng.integers(0, users, d)) for d in CRAFTED_INDEG]
    row_end = np.concatenate([np.zeros(users, np.uint64), np.cumsum(CRAFTED_INDEG).astype(np.uint64)])
    src = np.concatenate(s).astype(np.uint32)
    w = rng.integers(1, 6, len(src)).astype(np.int32)
    with L.LuxGraph.from_csc(row_end, src, w, app=L.APP_COLFILTER) as g:
        g.init()
        cf_wide_step(g, row_end, src, w, users, "crafted", min_wide=10)
