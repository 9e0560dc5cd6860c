"""Exact-arithmetic parity of the pull sweeps and of collaborative filtering, edge for edge.

The tolerance tests (1e-6 for PageRank, 2e-6 for CF) are wider than the effect of one dropped, duplicated or misrouted
edge into a large hub.  Here the kernels get inputs on which every summation order is exact (tests/graphs.py:
exact_pr_inputs, exact_cf_inputs), so the device must equal the oracle BIT FOR BIT whatever its reduction shape: one
`set_values` + `iterate(1)` against one oracle iteration from the same values, compared with np.array_equal.
tests/test_exact_method.py shows on the CPU that this comparison catches single wrong edges that the tolerances miss.

Covered, PageRank:
  * the plain flagged stream (seg.cuh), all 8 main shapes, on the small graphs and RMAT-17;
  * the forced source-blocked split (panel.cuh), all 6 panel shapes, at its edges: a block size that does not divide
    the hot set, a hot set smaller than one block (LUXB_HOT_MB), the 64-block cap, 32768-value blocks (15-bit
    offsets), every vertex a hub (min in-degree 1), (block, hub) pairs without edges;
  * both fix-ups (three kernels, LUXB_FUSED_FIXUP=0, and the fused chained scan) at RMAT-22 — more than 1024 fix-up
    blocks — over several set_values / iterate rounds on one handle (the chained scan's epochs are reused);
  * the merge-path tiles of pull.cuh, every LUXB_PULL_SHAPE, on device-resident and zero-copy edge arrays;
  * the default configuration at RMAT-22 and C1 (whole graph), and C2 on the oracle's destination blocks (heavy).
CC / SSSP through the forced panel split and the merge path: labels, iteration counts and traces bit-exact.
CF on a small bipartite graph and at C5 scale, one step each: the exact factors bit-exact, the others at 2e-6.
LUXB_SKIP_HEAVY=1 skips C2."""
import functools
import os

import numpy as np
import pytest

import oracle as O
import lux_b200 as L
from graphs import ALL_SMALL, exact_cf_inputs, exact_pr_inputs, in_degrees, rmat, symmetrize

pytestmark = pytest.mark.gpu
heavy = pytest.mark.skipif(os.environ.get("LUXB_SKIP_HEAVY") == "1", reason="LUXB_SKIP_HEAVY=1")
CF_GAMMA = np.float32(0.00000035)


@functools.lru_cache(maxsize=None)
def graph(name):
    """Host CSCs shared by the tests of this module (read only)."""
    if name in ALL_SMALL:
        return ALL_SMALL[name]()
    if name == "rmat16_sym":
        return symmetrize(*rmat(16, ef=8))
    return rmat(int(name[len("rmat"):]))


SMALL_AND_RMAT17 = sorted(ALL_SMALL) + ["rmat17"]


def set_env(monkeypatch, env):
    for k, v in env.items():
        monkeypatch.setenv(k, str(v))


def assert_bit_equal(gpu, ref, what):
    bad = np.nonzero(gpu.view(np.uint32) != ref.view(np.uint32))[0] if gpu.dtype == np.float32 else np.nonzero(gpu != ref)[0]
    assert bad.size == 0, "%s: %d values differ, first at %d: device %r, oracle %r" % (what, bad.size, bad[0], gpu[bad[0]], ref[bad[0]])


def exact_steps(g, row_end, src, what, rounds=1):
    """For every exact input x: set_values(x), iterate(1), and the result must be one oracle iteration from x, bit for
    bit.  rounds > 1 repeats with other values on the same handle."""
    nv = len(row_end)
    deg = O.out_degree(nv, src)
    max_in = int(in_degrees(row_end).max()) if len(src) else 0
    for r in range(rounds):
        for i, x in enumerate(exact_pr_inputs(nv, max_in, salt=r)):
            g.set_values(x)
            g.iterate(1)
            assert_bit_equal(g.values(), O.pagerank_iter(row_end, src, deg, x), "%s, round %d, input %d" % (what, r, i))


def run_exact(name, rounds=1, **kw):
    row_end, src = graph(name)
    with L.LuxGraph.from_csc(row_end, src, **kw) as g:
        g.init()
        st = g.stats()
        exact_steps(g, row_end, src, name, rounds)
    return st


def hot_set_size(row_end, src, hot_mb=24.0, cap=4096):
    """A second copy of the hot-set rule of build_hot_layout (lux_b200/csrc/api.cu): the vertices of out-degree >= tau,
    tau >= 2 the smallest threshold whose set fits in hot_mb MB of values (degrees clamped at 4096).  It must follow
    that function: it only serves to assert that each panel case below has the block count it is named after, and a
    drift shows up as a failed configuration assertion, not as a wrong value comparison."""
    nv = len(row_end)
    h_max = min(int(hot_mb * 1e6 / 4.0), nv)
    if h_max == 0 or nv < 2:
        return 0
    hist = np.bincount(np.minimum(O.out_degree(nv, src), cap), minlength=cap + 1)
    above = 0
    for d in range(cap, 1, -1):
        if above + int(hist[d]) > h_max:
            break
        above += int(hist[d])
    return above


# ---- 1. the plain flagged stream -------------------------------------------------------------------------------------
@pytest.mark.parametrize("main_shape", range(8))
def test_plain_seg_sweep_every_main_shape(main_shape, monkeypatch):
    set_env(monkeypatch, dict(LUXB_SB=0, LUXB_SEG_MAIN_SHAPE=main_shape))
    for name in SMALL_AND_RMAT17:
        assert run_exact(name)["panel_edges"] == 0


# ---- 2. the forced source-blocked split ------------------------------------------------------------------------------
# name: (graph, environment); LUXB_SB=1 forces the split, the rest sets its block size / cap / hub threshold / hot set
PANEL_EDGES = {
    "bs_not_dividing_the_hot_set": ("rmat16", dict(LUXB_SB_BS=1000, LUXB_SB_BLOCKS=48, LUXB_SB_MIN_INDEG=16)),
    "hot_set_smaller_than_one_block": ("rmat16", dict(LUXB_SB_BS=32768, LUXB_SB_BLOCKS=48, LUXB_SB_MIN_INDEG=8, LUXB_HOT_MB=0.02)),
    "64_blocks_cap": ("rmat16", dict(LUXB_SB_BS=128, LUXB_SB_BLOCKS=64, LUXB_SB_MIN_INDEG=4)),
    "bs_32768_15_bit_offsets": ("rmat17", dict(LUXB_SB_BS=32768, LUXB_SB_BLOCKS=48, LUXB_SB_MIN_INDEG=32)),
    "every_vertex_a_hub": ("rmat16", dict(LUXB_SB_BS=512, LUXB_SB_BLOCKS=48, LUXB_SB_MIN_INDEG=1)),
}


@pytest.mark.parametrize("panel_shape", range(6))
@pytest.mark.parametrize("case", sorted(PANEL_EDGES))
def test_panel_split_edges_every_panel_shape(case, panel_shape, monkeypatch):
    name, env = PANEL_EDGES[case]
    set_env(monkeypatch, dict(env, LUXB_SB=1, LUXB_SEG_PANEL_SHAPE=panel_shape, LUXB_SEG_MAIN_SHAPE=(panel_shape + 2) % 8))
    row_end, src = graph(name)
    hot = hot_set_size(row_end, src, float(env.get("LUXB_HOT_MB", 24.0)))
    bs, cap = env["LUXB_SB_BS"], env["LUXB_SB_BLOCKS"]
    st = run_exact(name)
    # the configuration is the one the case is named after
    assert st["panel_edges"] > 0 and st["panel_blocks"] == -(-min(hot, cap * bs) // bs), (st, hot)
    if case == "bs_not_dividing_the_hot_set":
        assert hot % bs != 0 and hot < cap * bs
    elif case == "hot_set_smaller_than_one_block":
        assert 0 < hot < bs and st["panel_blocks"] == 1
    elif case == "64_blocks_cap":
        assert st["panel_blocks"] == 64 and hot > 64 * bs
    elif case == "bs_32768_15_bit_offsets":
        assert hot > bs and st["panel_blocks"] == 2
    elif case == "every_vertex_a_hub":
        assert st["panel_hubs"] == int((in_degrees(row_end) > 0).sum())
        # fewer panel edges than (block, hub) pairs: some pairs have no edge (their slots stay at the identity)
        assert st["panel_edges"] < st["panel_hubs"] * st["panel_blocks"]


@pytest.mark.parametrize("panel_shape", range(6))
def test_panel_split_small_graphs_every_panel_shape(panel_shape, monkeypatch):
    """Tiny blocks and hub threshold on the small graphs: hubs spanning pieces in both streams, hubs whose edges all
    moved to the panel, graphs without edges or without a hot set (the split then stays off)."""
    set_env(monkeypatch, dict(LUXB_SB=1, LUXB_SB_BS=16, LUXB_SB_MIN_INDEG=2, LUXB_SB_BLOCKS=48, LUXB_SEG_PANEL_SHAPE=panel_shape))
    for name in sorted(ALL_SMALL):
        run_exact(name)


# ---- 3. both fix-ups at RMAT-22, several rounds on one handle ---------------------------------------------------------
@functools.lru_cache(maxsize=1)
def rmat22():
    scale = 22
    return O.gen_rmat_csc(scale, 1 << scale, 16 << scale, 27)


@pytest.mark.parametrize("fused", [0, 1])
@pytest.mark.parametrize("layout", ["plain", "default"])
def test_fixups_rmat22_several_rounds(layout, fused, monkeypatch):
    """plain: the whole graph in one stream of 256-edge pieces, 2048-edge stages (main shape 6); 2^26 edges plus one
    stage of padding make 262 152 pieces, 1025 fix-up blocks, so the three-kernel fix-up's block scan runs serial
    chunks of two.  default: the automatic split (panel + main, two fix-ups per sweep).  Three rounds of set_values /
    iterate on one handle reuse the chained scan's status words."""
    env = dict(LUXB_FUSED_FIXUP=fused)
    if layout == "plain":
        env.update(LUXB_SB=0, LUXB_SEG_MAIN_SHAPE=6)
    set_env(monkeypatch, env)
    row_end, src = rmat22()
    if layout == "plain":  # the reason this runs at RMAT-22: more fix-up blocks than the block scan has threads
        stage, piece, fix_block = 2048, 256, 256
        n_pieces = (len(src) // stage + 1) * (stage // piece)  # the stream is padded with 1 .. stage dummy words
        assert -(-n_pieces // fix_block) > 1024
    scale = 22
    with L.LuxGraph.from_rmat(scale, 1 << scale, 16 << scale, 27) as g:
        g.init()
        st = g.stats()
        assert (st["panel_edges"] > 0) == (layout == "default")
        exact_steps(g, row_end, src, "rmat22 %s fused=%d" % (layout, fused), rounds=3)


# ---- 4. the merge path -------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("zero_copy", [False, True])
@pytest.mark.parametrize("pull_shape", [0, 1, 2])
def test_merge_path_every_pull_shape(pull_shape, zero_copy, monkeypatch):
    """LUXB_SWEEP=merge on device-resident edges; zero-copy graphs keep their edges in mapped host memory and always
    take the merge path."""
    env = dict(LUXB_PULL_SHAPE=pull_shape)
    if not zero_copy:
        env["LUXB_SWEEP"] = "merge"
    set_env(monkeypatch, env)
    for name in SMALL_AND_RMAT17:
        assert run_exact(name, zero_copy=zero_copy)["panel_edges"] == 0


# ---- 5. the default configuration at scale ----------------------------------------------------------------------------
def test_default_c1_whole_graph():
    nv, ne, seed = 7414866, 194109311, 1
    with L.LuxGraph.from_rmat(23, nv, ne, seed) as g:
        row_end, src = g.local_csc()
        g.init()
        exact_steps(g, row_end, src, "C1")


@heavy
def test_default_c2_rmat27_oracle_blocks():
    """RMAT-27: hubs with up to 1.3 M in-edges, so K = 1 — a counting pass of ones, then source-bit passes.  Compared
    on the oracle generator's destination blocks (hubs, pseudo-random blocks, the tail)."""
    scale, seed = 27, 27
    nv, ne = 1 << scale, 16 << scale
    block_shift = 14
    nb = nv >> block_shift
    sel = (np.random.default_rng(7).integers(0, 32, nb) == 0).astype(np.uint8)
    sel[0] = sel[1] = sel[nb - 1] = 1
    blk = O.rmat_blocks(scale, nv, ne, seed, block_shift, sel, want_deg=True)
    max_in = int(in_degrees(blk["row_end"]).max())
    xs = exact_pr_inputs(nv, max_in, passes=3)
    assert len(xs) == 3  # the top hub (vertex block 0) is sampled: K = 1
    with L.LuxGraph.from_rmat(scale, nv, ne, seed) as g:
        g.init()
        assert g.stats()["panel_edges"] > 0
        assert np.array_equal(g.out_degree(), blk["deg"])
        for i, x in enumerate(xs):
            g.set_values(x)
            g.iterate(1)
            got = g.values()[blk["vid"]]
            assert_bit_equal(got, O.pagerank_iter_compact(nv, blk, blk["deg"], x), "C2 input %d" % i)


# ---- 6. CC / SSSP pull iterations through the panel split and the merge path ----------------------------------------
LABEL_PATHS = {
    "panel_small_blocks": dict(LUXB_SB=1, LUXB_SB_BS=64, LUXB_SB_MIN_INDEG=2, LUXB_SB_BLOCKS=48, LUXB_SEG_PANEL_SHAPE=0),
    "panel_every_hub_64_blocks": dict(LUXB_SB=1, LUXB_SB_BS=128, LUXB_SB_MIN_INDEG=1, LUXB_SB_BLOCKS=64, LUXB_SEG_PANEL_SHAPE=5),
    "merge": dict(LUXB_SWEEP="merge"),
}
LABEL_RUNS = [("cc", "rmat16_sym", 0), ("cc", "two_components", 0), ("cc", "star", 0), ("cc", "trailing_isolated", 0),
              ("sssp", "rmat16", 0), ("sssp", "rmat16", 12345), ("sssp", "star", 0), ("sssp", "chain", 0)]


@pytest.mark.parametrize("path", sorted(LABEL_PATHS))
def test_labels_through_panel_and_merge_paths(path, monkeypatch):
    set_env(monkeypatch, LABEL_PATHS[path])
    for app_name, name, start in LABEL_RUNS:
        app, oapp = (L.APP_CC, O.APP_CC) if app_name == "cc" else (L.APP_SSSP, O.APP_SSSP)
        row_end, src = graph(name)
        what = "%s %s start %d" % (app_name, name, start)
        with L.LuxGraph.from_csc(row_end, src, app=app, start=start) as g:
            g.init()
            st = g.stats()
            it = g.run_to_convergence()
            lab = g.values()
            bad = g.check()
            active, pull = g.trace()
        ref = O.label_run(oapp, row_end, src, P=1, start=start)
        assert np.array_equal(lab, ref["labels"]), what
        assert bad == 0 and it == ref["iters"], what
        assert np.array_equal(active, ref["active"]) and np.array_equal(pull, ref["pull"]), what
        if name.startswith("rmat"):
            assert pull.any(), what  # the sweep under test ran
            assert (st["panel_edges"] > 0) == path.startswith("panel"), (what, st)


# ---- 7. collaborative filtering ----------------------------------------------------------------------------------------
def cf_exact_step(g, row_end, src, w, users, items, what):
    x = exact_cf_inputs(users, items, int(in_degrees(row_end)[users:].max()))
    g.set_values(x)
    g.iterate(1)
    gpu = g.values()
    ref = O.cf_iter(row_end, src, w, x)
    exact = ref[users:, 10:]
    assert np.abs(exact).max() / CF_GAMMA < (1 << 22) * (1 - 1e-6), "accumulators too large to be exact"
    assert np.count_nonzero(exact) > 0.9 * exact.size  # items with in-edges: the exact factors carry the sums
    assert_bit_equal(gpu[users:, 10:].reshape(-1), exact.reshape(-1), what + ", items' factors 10-19")
    assert np.allclose(gpu, ref, rtol=2e-6, atol=0), what


def test_colfilter_small_bipartite_exact():
    users, items = 300, 40
    row_end, src, w = O.gen_bipartite_csc(users, items, 20000, 5)
    with L.LuxGraph.from_csc(row_end, src, w, app=L.APP_COLFILTER) as g:
        g.init()
        cf_exact_step(g, row_end, src, w, users, items, "small bipartite")


def test_colfilter_c5_scale_exact():
    users, items, ratings, seed = 480189, 17770, 100480507, 5
    with L.LuxGraph.from_bipartite(users, items, ratings, seed) as g:
        row_end, src, w = g.local_csc(weighted=True)
        g.init()
        cf_exact_step(g, row_end, src, w, users, items, "C5")
